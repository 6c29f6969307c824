// percentile_doy: day-of-year rolling-window percentiles per grid cell.
//
// Replaces core/calendar.py:395-494 (`percentile_doy`: rolling(center).construct -> unstack by
// (year, dayofyear) -> stack (year, window) -> calc_perc) and core/utils.py:279-557 (the NaN-aware
// Hyndman-Fan quantile with its full sort, :538).
//
// Sample of day-of-year d (window w = 2h+1):  S(d) = { x[i+k] : doy(i) = d, |k| <= h, 0 <= i+k < T }.
//
// Design.  The (time, lat, lon) buffer is coalesced along cells, so a LANE owns one cell
// (a warp reads one 128-byte row segment per time step) and keeps the order statistics it needs in
// REGISTERS: only the K extreme values of S(d) matter (K = 16 for the 90th percentile of 150
// samples), never the full sort the reference does.
//   * generic kernel (any calendar): a small (year, doy) -> row table drives direct insertion of
//     every sample into a sorted K-register list (2K min/max per sample).
//   * fast kernel (all years the same length, e.g. noleap / 360_day): S(d) is the union of the w
//     per-day lists Y(e) = { x[y*L + e] : y }, e = d-h..d+h.  Each Y(e) is loaded once (N coalesced
//     rows), sorted by a register sorting network and kept for the w consecutive days that use
//     it; S(d)'s K extremes come from w-1 bitonic top-K merges.  Days are processed in order so
//     every input row is read once per chunk (+2h halo days).
// No shared memory, no tensor cores (there is no contraction); the kernel is bound by the
// min/max (ALU) pipe, see DESIGN.md.
#include <cuda.h>   // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)

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

__device__ __forceinline__ void store_vec4(int32_t* dst, const int32_t (&v)[4]) {
  *reinterpret_cast<int4*>(dst) = make_int4(v[0], v[1], v[2], v[3]);
}

// value as inserted in the lists: NaN -> -inf (never selected), bottom side -> negated
__device__ __forceinline__ float prep(float v, bool top, int& n) {
  const bool ok = (v == v);
  n += ok ? 1 : 0;
  v = top ? v : -v;
  return ok ? v : XC_NEG_INF;
}

template <int K>
__device__ __forceinline__ void insert_desc(float (&lst)[K], float v) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float hi = fmaxf(lst[k], v);
    v = fminf(lst[k], v);
    lst[k] = hi;
  }
}

// ------------------------------------------------------------------------------------------------
// generic kernel: pos[y * n_doy + (d-1)] = row of (year y, doy d) or -1
// ------------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(kThreads)
percentile_doy_generic_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                              const int32_t* __restrict__ pos, int32_t n_doy, int32_t n_years, int32_t h,
                              QuantSpec spec, int32_t doys_per_chunk, double* __restrict__ out,
                              int32_t d_begin, int32_t d_end, const int32_t* __restrict__ vrow) {
  const int64_t c = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (c >= C) return;
  const int d0 = d_begin + blockIdx.y * doys_per_chunk;
  const int d1 = min(d_end, d0 + doys_per_chunk);
  const float* col = x + c;
  const bool top = spec.top != 0;
  for (int d = d0; d < d1; ++d) {
    float lst[K];
#pragma unroll
    for (int k = 0; k < K; ++k) lst[k] = XC_NEG_INF;
    int n = 0;
    for (int y = 0; y < n_years; ++y) {
      const int i = pos[y * n_doy + d];
      if (i < 0) continue;
      const int j0 = max(0, i - h), j1 = min((int)T - 1, i + h);
      for (int j = j0; j <= j1; ++j) {
        // vrow: the row holding the value of (virtual) step j, -1 = missing (bootstrap replacements)
        const int row = vrow ? vrow[j] : j;
        if (row < 0) continue;
        const float v = prep(__ldg(col + (int64_t)row * ldx), top, n);
        insert_desc<K>(lst, v);
      }
    }
    out[(int64_t)d * C + c] = finalize_quantile<K>(lst, n, spec);
  }
}

// ------------------------------------------------------------------------------------------------
// selection kernel: percentiles whose order statistics lie more than 64 ranks from both ends of the
// sample (e.g. the median of 30 x 5 values).  A lane owns one cell: the non-NaN values of the day's
// sample go to the lane's shared-memory column as order-preserving integer keys, the k-th smallest
// is built bit by bit (v = max{t : #{key < t} <= k}, 32 counting passes), its successor is the
// smallest key above it unless ties already cover rank k+1.  Exact for any sample that fits shared
// memory (n_years * window <= 768); ~30x the cost of the network kernels, used only when needed.
// ------------------------------------------------------------------------------------------------
constexpr int kSelThreads = 64;

__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__global__ void __launch_bounds__(kSelThreads)
percentile_doy_select_kernel(const float* __restrict__ x, int64_t T, int64_t C, int64_t ldx,
                             const int32_t* __restrict__ pos, int32_t n_doy, int32_t n_years, int32_t h,
                             QuantSpec spec, int32_t doys_per_chunk, double* __restrict__ out,
                             const int32_t* __restrict__ vrow) {
  extern __shared__ uint32_t keys[];  // [n_years * (2h+1)][kSelThreads]
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kSelThreads + lane;
  if (c >= C) return;
  const int d0 = blockIdx.y * doys_per_chunk;
  const int d1 = min(n_doy, d0 + doys_per_chunk);
  const float* col = x + c;
  uint32_t* mine = keys + lane;
  for (int d = d0; d < d1; ++d) {
    int n = 0;
    for (int y = 0; y < n_years; ++y) {
      const int i = pos[y * n_doy + d];
      if (i < 0) continue;
      const int j0 = max(0, i - h), j1 = min((int)T - 1, i + h);
      for (int j = j0; j <= j1; ++j) {
        const int row = vrow ? vrow[j] : j;
        if (row < 0) continue;
        const float v = __ldg(col + (int64_t)row * ldx);
        if (v == v) mine[(n++) * kSelThreads] = order_key(v);
      }
    }
    double res;
    if (n == 0) {
      res = __longlong_as_double(0x7ff8000000000000LL);
    } else {
      const QuantIdx qi = quant_index(n, spec);
      // rank of the left neighbour: clamps of core/utils.py:417-461 (vi >= n-1 -> max, vi < 0 -> min)
      int k = qi.ilo;
      bool single = (n == 1);
      if (n > 1 && qi.vi >= (double)n - 1.0) { k = n - 1; single = true; }
      if (n > 1 && qi.vi < 0.0) { k = 0; single = true; }
      if (n == 1) k = 0;
      uint32_t v = 0u;
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t t = v | (1u << bit);
        int cnt = 0;
        for (int i = 0; i < n; ++i) cnt += (mine[i * kSelThreads] < t) ? 1 : 0;
        v = (cnt <= k) ? t : v;
      }
      const float left = key_value(v);
      if (single) {
        res = (double)left;
      } else {
        int le = 0;
        uint32_t nxt = 0xffffffffu;
        for (int i = 0; i < n; ++i) {
          const uint32_t q = mine[i * kSelThreads];
          le += (q <= v) ? 1 : 0;
          nxt = (q > v && q < nxt) ? q : nxt;
        }
        const float right = (le >= k + 2) ? left : key_value(nxt);
        res = quant_lerp(left, right, qi);
      }
    }
    out[(int64_t)d * C + c] = res;
  }
}

#ifndef XC_PCTL_VARIANT
#define XC_PCTL_VARIANT 0
#endif
#ifndef XC_PCTL_ADDR      // 0: running 64-bit pointer (2 ALU-pipe adds per load); 1: one IMAD.WIDE (FMA pipe)
#define XC_PCTL_ADDR (XC_PCTL_VARIANT == 1 ? 1 : 0)
#endif
#ifndef XC_PCTL_STAGE     // 1: cp.async staging of the next day's rows in the window-5 paired kernel
#define XC_PCTL_STAGE 1      // (an L2 prefetch of those rows was slower)
#endif
#ifndef XC_PCTL_PROBE     // NaN probe: 0 = compare chain (ALU pipe); 1 = FMA chain; 2 = FADD tree + 1 compare per 4
#define XC_PCTL_PROBE (XC_PCTL_VARIANT == 1 ? 1 : 0)
#endif

// NV rows p0 + k*ystride -> v[0..NV)
template <int K, int NV>
__device__ __forceinline__ void fetch_rows(const char* p0, uint64_t ystride, float (&v)[K]) {
#if XC_PCTL_ADDR == 1
  const uint32_t ys32 = (uint32_t)ystride;
#pragma unroll
  for (int k = 0; k < NV; ++k)
    v[k] = ld_stream(reinterpret_cast<const float*>(p0 + (uint64_t)((uint32_t)k) * (uint64_t)ys32));
#else
  const char* pp = p0;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    v[k] = ld_stream(reinterpret_cast<const float*>(pp));
    pp += ystride;
  }
#endif
}

// v[0..NV) raw values -> negated for a bottom-side quantile, pads -inf, NaN -> -inf (never selected;
// nv counts the valid ones), sorted descending.
template <int K, int NV>
__device__ __forceinline__ void finish_chunk(bool top, float (&v)[K], int& nv) {
#pragma unroll
  for (int k = NV; k < K; ++k) v[k] = XC_NEG_INF;
  if (!top) {
#pragma unroll
    for (int k = 0; k < NV; ++k) v[k] = -v[k];
  }
  // NaN handling off the fast path: only a lane that may hold a NaN looks at each value
#if XC_PCTL_PROBE == 1
  float probe = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) probe = __fmaf_rn(v[k], 0.f, probe);
  const bool suspicious = (probe != probe);
#elif XC_PCTL_PROBE == 2
  // sums of four on the FMA pipe: NaN iff a NaN (or +inf and -inf) is among them
  bool suspicious = false;
#pragma unroll
  for (int k = 0; k < NV; k += 4) {
    float a = v[k];
    if (k + 1 < NV) a = __fadd_rn(a, v[k + 1]);
    float b = (k + 2 < NV) ? v[k + 2] : 0.f;
    if (k + 3 < NV) b = __fadd_rn(b, v[k + 3]);
    const float q = __fadd_rn(a, b);
    suspicious = suspicious || (q != q);
  }
#else
  bool suspicious = false;
#pragma unroll
  for (int k = 0; k < NV; ++k) suspicious = suspicious || (v[k] != v[k]);
#endif
  nv = NV;
  if (suspicious) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const bool bad = (v[k] != v[k]);
      nv -= bad ? 1 : 0;
      v[k] = bad ? XC_NEG_INF : v[k];
    }
  }
  if constexpr (NV == K) sort_desc<K>(v);
  else sort_desc_first<K, NV>(v);
}

template <int K, int NV>
__device__ __forceinline__ void load_sort_chunk(const char* p0, uint64_t ystride, bool top, float (&v)[K],
                                                int& nv) {
  fetch_rows<K, NV>(p0, ystride, v);
  finish_chunk<K, NV>(top, v, nv);
}

// ---- asynchronous staging of the NEXT day's rows (cp.async, global -> shared) --------------------
// The day-list kernels are bound by the min/max pipe but lose a third of their issue slots waiting
// for the 30 row loads of a day (long-scoreboard stalls).  With a Stager the rows of day e+1 are
// copied to a per-lane shared-memory column while day e is sorted and merged; a lane reads back only
// what it copied itself, so cp.async.wait_group is the only synchronisation.  The buffer is reused
// chunk by chunk: as soon as the 16 (14) values of a chunk are in registers, the copy of the same
// chunk of the next day is issued, so that exactly two groups are pending at the start of a day.
// Used when a day has two chunks with every year present (K == 16, 30..32 years, 0 <= e < L).
struct Stager {
  float* col;      // this lane's column of the [32][kThreads] staging buffer
  int staged_e;    // day in flight / in the buffer, or kNoDay
  bool want_next;  // the caller asks for day e + 1 next
};
constexpr int kNoDay = -1000000;

__device__ __forceinline__ void cp_async4(float* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// chunk of NV years starting at year y0 of day e: from the staging buffer (have) or from global;
// then (issue) start the copy of the same chunk of day e + 1
template <int K, int NV>
__device__ __forceinline__ void staged_chunk(Stager& sg, const char* pcur, uint64_t ystride, int64_t day_bytes,
                                             int y0, bool have, bool issue, bool top, float (&v)[K], int& nv) {
  if (have) {
    if (issue) cp_async_wait<1>(); else cp_async_wait<0>();
#pragma unroll
    for (int k = 0; k < NV; ++k) v[k] = sg.col[(y0 + k) * kThreads];
  } else {
    fetch_rows<K, NV>(pcur + (uint64_t)y0 * ystride, ystride, v);
  }
  if (issue) {
    const char* pn = pcur + day_bytes + (uint64_t)y0 * ystride;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      cp_async4(sg.col + (y0 + k) * kThreads, pn);
      pn += ystride;
    }
    cp_async_commit();
  }
  finish_chunk<K, NV>(top, v, nv);
}

// ------------------------------------------------------------------------------------------------
// fast kernel: uniform year length L == n_doy, T == N*L, series starts on doy 1
// ------------------------------------------------------------------------------------------------
// Sorted (descending) K extremes of Y(e) = { x[y*L + e] : 0 <= y*L + e < T } ; e may lie in
// [-h, L+h) (the window reaches into the neighbouring year, core/calendar.py:448 pads only at the
// two ends of the SERIES).
// Table mode (pos != nullptr; calendars whose years differ in length): the row of (year y, day e) is
// pos[y * n_doy + e] (-1 when that day does not exist); only days e in [0, n_doy) are requested.
template <int K, bool TABLE = false>
__device__ __forceinline__ void load_day_list(const float* __restrict__ x, int64_t c, int64_t ldx, int T, int L,
                                              int N, int e, bool top, float (&lst)[K], int& n,
                                              const int32_t* __restrict__ pos = nullptr, int n_doy = 0,
                                              Stager* sg = nullptr) {
  n = 0;
  if constexpr (TABLE) {
    bool first_t = true;
    for (int y0 = 0; y0 < N; y0 += K) {
      float v[K];
      int nv = 0;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int y = y0 + k;
        const int row = (y < N) ? pos[y * n_doy + e] : -1;
        float r = XC_NEG_INF;
        if (row >= 0) {
          r = ld_stream(x + (int64_t)row * ldx + c);
          const bool ok = (r == r);
          nv += ok ? 1 : 0;
          r = ok ? (top ? r : -r) : XC_NEG_INF;
        }
        v[k] = r;
      }
      n += nv;
      sort_desc<K>(v);
      if (first_t) {
#pragma unroll
        for (int k = 0; k < K; ++k) lst[k] = v[k];
        first_t = false;
      } else {
        merge_top_desc<K>(lst, v);
      }
    }
    return;
  }
  // rows y*L + e that exist: e < 0 reaches into the previous year (no year -1), e >= L into the next
  const int ylo = (e < 0) ? 1 : 0;
  const int yhi = (e >= L) ? N - 1 : N;
  const uint64_t ystride = (uint64_t)L * (uint64_t)ldx * 4ull;
  const bool narrow = (ystride >> 32) == 0;
  if constexpr (K == 16) {
    if (sg != nullptr) {
      const int tail2 = N - K;                                   // years in the second chunk
      const bool two_chunks = narrow && tail2 >= 14 && tail2 <= 16;
      const bool now_ok = two_chunks && e >= 0 && e < L;         // every year has day e
      if (now_ok) {
        const bool have = (sg->staged_e == e);
        const bool issue = sg->want_next && (e + 1 < L);
        const char* pcur = reinterpret_cast<const char*>(x + (int64_t)e * ldx + c);
        const int64_t day_bytes = ldx * 4;
        float v[K];
        int nv;
        staged_chunk<K, K>(*sg, pcur, ystride, day_bytes, 0, have, issue, top, lst, nv);
        n = nv;
        if (tail2 == 14) staged_chunk<K, 14>(*sg, pcur, ystride, day_bytes, K, have, issue, top, v, nv);
        else if (tail2 == 15) staged_chunk<K, 15>(*sg, pcur, ystride, day_bytes, K, have, issue, top, v, nv);
        else staged_chunk<K, 16>(*sg, pcur, ystride, day_bytes, K, have, issue, top, v, nv);
        n += nv;
        merge_top_desc<K>(lst, v);
        sg->staged_e = issue ? e + 1 : kNoDay;
        return;
      }
      // a day that cannot be staged is never announced by the previous one (same predicate), so
      // nothing is in flight here
      sg->staged_e = kNoDay;
    }
  }
  bool first = true;
  for (int y0 = 0; y0 < N; y0 += K) {
    float v[K];
    int nv;
    // byte address of (row (y0+k)*L + e, cell c) = p0 + k * ystride
    const char* p0 = reinterpret_cast<const char*>(x + ((int64_t)y0 * L + e) * ldx + c);
    const int tail = N - y0;  // warp-uniform
    const bool inside = narrow && (y0 >= ylo) && ((tail >= K ? y0 + K : N) <= yhi);
    // The last chunk of e.g. a 30-year base holds 14 values + 2 pads (-inf, already at the bottom):
    // its loads are unconditional and comparators touching the padded wires are left out.
    if (inside && tail >= K) {
      load_sort_chunk<K, K>(p0, ystride, top, v, nv);
    } else if (K == 16 && inside && tail == 14) {
      load_sort_chunk<K, (K == 16 ? 14 : K)>(p0, ystride, top, v, nv);
    } else if (K == 16 && inside && tail == 15) {
      load_sort_chunk<K, (K == 16 ? 15 : K)>(p0, ystride, top, v, nv);
    } else {
      nv = 0;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int y = y0 + k;
        const bool ok = (y >= ylo) && (y < yhi);
        float r = ok ? ld_stream(reinterpret_cast<const float*>(p0 + (uint64_t)k * ystride)) : XC_NEG_INF;
        const bool good = ok && (r == r);
        nv += good ? 1 : 0;
        v[k] = good ? (top ? r : -r) : XC_NEG_INF;
      }
      sort_desc<K>(v);
    }
    n += nv;
    if (first) {
#pragma unroll
      for (int k = 0; k < K; ++k) lst[k] = v[k];
      first = false;
    } else {
      merge_top_desc<K>(lst, v);
    }
  }
}

// Per-lane ring of the W-1 most recent day lists in SHARED memory, laid out [slot][k][lane] so that
// a warp's access to element k of a slot is one conflict-free 128-byte wavefront (each lane only
// ever touches its own column).  Keeping the ring out of the register file lets ~24 warps per SM
// stay resident (the kernel is latency-bound otherwise) and keeps the code small enough for the
// instruction cache (one copy of the sorting network and of the merge, no unrolling over W).
template <int K, bool TABLE>
__global__ void __launch_bounds__(kThreads)
percentile_doy_uniform_kernel(const float* __restrict__ x, int32_t T, int64_t C, int64_t ldx, int32_t L,
                              int32_t N, int32_t W, QuantSpec spec, int32_t doys_per_chunk,
                              double* __restrict__ out, const int32_t* __restrict__ pos, int32_t n_doy,
                              int32_t d_begin, int32_t d_end) {
  extern __shared__ float smem[];
  const int H = W / 2;
  const int R = W - 1;  // ring slots
  float* ring = smem;                                        // [R][K][kThreads]
  int* rcnt = reinterpret_cast<int*>(smem + (size_t)R * K * kThreads);  // [R][kThreads]
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kThreads + lane;
  if (c >= C) return;  // no block-level synchronisation below: every lane owns its smem column
  const int d0 = d_begin + blockIdx.y * doys_per_chunk;
  const int d1 = min(d_end, d0 + doys_per_chunk);
  if (d0 >= d1) return;
  const bool top = spec.top != 0;

  float ynew[K];
  int nnew;
  // prologue: day lists e = d0-H .. d0+H-1 -> ring slots 0..R-1 (slot = (e - (d0-H)) mod R)
  for (int s = 0; s < R; ++s) {
    load_day_list<K, TABLE>(x, c, ldx, T, L, N, d0 - H + s, top, ynew, nnew, pos, n_doy);
#pragma unroll
    for (int k = 0; k < K; ++k) ring[((size_t)s * K + k) * kThreads + lane] = ynew[k];
    rcnt[s * kThreads + lane] = nnew;
  }
  int oldest = 0;  // slot holding day list e = d-H
  for (int d = d0; d < d1; ++d) {
    load_day_list<K, TABLE>(x, c, ldx, T, L, N, d + H, top, ynew, nnew, pos, n_doy);
    float acc[K];
#pragma unroll
    for (int k = 0; k < K; ++k) acc[k] = ynew[k];
    int n = nnew;
#pragma unroll 1
    for (int s = 0; s < R; ++s) {
      const float* slot = ring + (size_t)s * K * kThreads + lane;
      // acc <- top-K of (acc U slot): max against the reversed list, then bitonic clean-up
#pragma unroll
      for (int k = 0; k < K; ++k) acc[k] = fmaxf(acc[k], slot[(size_t)(K - 1 - k) * kThreads]);
      bitonic_finish_desc<K>(acc);
      n += rcnt[s * kThreads + lane];
    }
    out[(int64_t)d * C + c] = finalize_quantile<K>(acc, n, spec);
    // the new list replaces the oldest one
#pragma unroll
    for (int k = 0; k < K; ++k) ring[((size_t)oldest * K + k) * kThreads + lane] = ynew[k];
    rcnt[oldest * kThreads + lane] = nnew;
    oldest = (oldest + 1 == R) ? 0 : oldest + 1;
  }
}

// float32 threshold t32 with (x op t32) == ((double)x op t) for every float32 x (directed rounding)
template <int OP>
__device__ __forceinline__ float fold_thr(double t) {
  float f = __double2float_rn(t);
  if (t != t) return f;  // NaN threshold: every compare is False
  if constexpr (OP == XC_OP_GT || OP == XC_OP_LE) {  // largest float32 <= t
    if ((double)f > t) f = __int_as_float(__float_as_int(f) + ((f > 0.f) ? -1 : 1));
    if (f == 0.f && t < 0.0) f = -1.401298464e-45f;
  } else {                                           // smallest float32 >= t
    if ((double)f < t) f = __int_as_float(__float_as_int(f) + ((f >= 0.f) ? 1 : -1));
    if (f == 0.f && t > 0.0) f = 1.401298464e-45f;
  }
  return f;
}


#ifndef XC_PCTL_PAIR_MINBLOCKS   // with the staging buffer 4 CTAs fit an SM (51 KB each)
#define XC_PCTL_PAIR_MINBLOCKS 4
#endif
// (A day-by-day window-5 kernel with the fused per-year count of the same series -- tx90p sub-case 3a in one
// pass -- was slower than the two-kernel path and was removed.)
// Window 5, days handled in PAIRS.  With B(d) = Y(d-2..d+1) = A(d-1) U A(d+1) the windows of two
// neighbouring days are one rank-only merge away:  S(d-1) = Y(d-3) U B(d)  and  S(d) = B(d) U Y(d+2).
// Per pair of days: one pair merge A(d+1), one merge B(d), two rank-only finals (2*80 + 2*32
// min/max) instead of 2*(80 + 80 + 32) for the day-by-day kernel above; the per-day sort of the N
// values of a day (the larger part of the work) is unchanged.
// The loop still advances ONE day per iteration (even/odd branch) so that the body holds a single
// copy of the day-list sort and of the final merge: two inlined copies overflow the 32 KB
// instruction cache and cost more than the saved merges.
// Shared memory per lane: A(d-1), the two most recent odd-position day lists Y(d-3), Y(d-1), and
// the even-position list Y(d) waiting for its partner.
template <int K, bool TABLE>
__global__ void __launch_bounds__(kThreads, XC_PCTL_PAIR_MINBLOCKS)
percentile_doy_w5p_kernel(const float* __restrict__ x, int32_t T, int64_t C, int64_t ldx, int32_t L, int32_t N,
                          QuantSpec spec, int32_t doys_per_chunk, double* __restrict__ out,
                          const int32_t* __restrict__ pos, int32_t n_doy, int32_t d_begin, int32_t d_end) {
  extern __shared__ float smem[];
  float* sA = smem;                                                    // [K][kThreads]
  float* sY = smem + (size_t)K * kThreads;                             // [2][K][kThreads]
  float* sE = smem + (size_t)3 * K * kThreads;                         // [K][kThreads]
  int* sn = reinterpret_cast<int*>(smem + (size_t)4 * K * kThreads);   // [4][kThreads]: n(A), n(Y0), n(Y1), n(E)
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kThreads + lane;
  if (c >= C) return;
  const int p0 = d_begin + blockIdx.y * doys_per_chunk;
  const int p1 = min(d_end, p0 + doys_per_chunk);
  if (p0 >= p1) return;
  const bool top = spec.top != 0;

  auto store_list = [&](float* dst, const float (&a)[K]) {
#pragma unroll
    for (int k = 0; k < K; ++k) dst[(size_t)k * kThreads + lane] = a[k];
  };

  float t[K], ynew[K], o[K];
  int nnew, nB = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) t[k] = 0.f;
#if XC_PCTL_STAGE
  Stager stager{reinterpret_cast<float*>(sn + 4 * kThreads) + lane, kNoDay, false};
  Stager* sg = (K == 16 && !TABLE) ? &stager : nullptr;
#else
  Stager* sg = nullptr;
#endif
  // The four warm-up iterations day = p0-4 .. p0-1 run the steady-state code without emitting:
  // they leave Y(p0-2), Y(p0) in the two odd slots, A(p0) = Y(p0-1) U Y(p0) in sA and Y(p0+1) in sE
  // (what they compute from the not-yet-written lists is overwritten before it is used).  No
  // separate prologue means one copy of the day-list sort in the whole kernel.
  int s = 0;  // slot of Y(d-3)
#pragma unroll 1
  for (int day = p0 - 4; day < p1; ++day) {
    if (sg) sg->want_next = (day + 1 < p1);
    load_day_list<K, TABLE>(x, c, ldx, T, L, N, day + 2, top, ynew, nnew, pos, n_doy, sg);
    int n;
    if (((day - p0) & 1) == 0) {
      // first day of the pair (day = d-1): ynew = Y(d+1)
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = fmaxf(sE[(size_t)k * kThreads + lane], ynew[K - 1 - k]);
      bitonic_finish_desc<K>(o);       // o <- A(d+1)
      const int nA1 = sn[3 * kThreads + lane] + nnew;
#pragma unroll
      for (int k = 0; k < K; ++k) t[k] = fmaxf(sA[(size_t)k * kThreads + lane], o[K - 1 - k]);
      bitonic_finish_desc<K>(t);       // t <- B(d)
      nB = sn[lane] + nA1;
      store_list(sA, o);
      sn[lane] = nA1;
      float* slot = sY + (size_t)s * K * kThreads;
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = slot[(size_t)k * kThreads + lane];   // Y(d-3)
      n = nB + sn[(1 + s) * kThreads + lane];
      store_list(slot, ynew);          // Y(d+1) replaces Y(d-3)
      sn[(1 + s) * kThreads + lane] = nnew;
      s ^= 1;
    } else {
      // second day of the pair (day = d): ynew = Y(d+2), the even-position list of the next pair
      store_list(sE, ynew);
      sn[3 * kThreads + lane] = nnew;
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = ynew[k];
      n = nB + nnew;
    }
    if (day < p0) continue;
    // quantile of (t U o), both sorted descending, n valid values in the window
    float u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = fmaxf(t[k], o[K - 1 - k]);
    const QuantIdx qi = quant_index(n, spec);
    const bool in_range = (n >= 2) && (qi.vi < (double)n - 1.0) && (qi.vi >= 0.0);
    const bool fast = in_range && (top ? (n - 1 - qi.ilo == K - 1) : (qi.ilo + 1 == K - 1));
    double res;
    if (__all_sync(__activemask(), fast)) {
      // only the two smallest of the bitonic top-K are needed
      float m[K / 2];
#pragma unroll
      for (int i = 0; i < K / 2; ++i) m[i] = fminf(u[i], u[i + K / 2]);
#pragma unroll
      for (int h = K / 4; h >= 2; h >>= 1) {
#pragma unroll
        for (int i = 0; i < h; ++i) m[i] = fminf(m[i], m[i + h]);
      }
      const float smallest = fminf(m[0], m[1]), second = fmaxf(m[0], m[1]);
      res = top ? quant_lerp(smallest, second, qi) : quant_lerp(-second, -smallest, qi);
    } else {
      bitonic_finish_desc<K>(u);
      res = finalize_quantile<K>(u, n, spec);
    }
    out[(int64_t)day * C + c] = res;
  }
}


// ------------------------------------------------------------------------------------------------
// Window 5, paired days, rows delivered by TMA (sm_90a: cp.async.bulk.tensor + mbarrier).
//
// Same arithmetic as percentile_doy_w5p_kernel (identical networks, identical results), but the N
// rows of a day-of-year are no longer fetched lane by lane (N loads, 2 N 64-bit address adds on the
// min/max pipe, N cp.async issue slots per lane and day): the input is described ONCE as a 3-D tensor
// (cell, day-of-year, year) and a dedicated producer warp issues ONE bulk tensor copy per day --
// box 128 cells x 1 day x N years -> the [N][128] staging tile -- against an mbarrier; the four
// consumer warps only wait, read their column (conflict-free LDS) and run the networks.  A window
// day that reaches into the neighbouring year is the same box shifted by one year: the year that
// does not exist is OUT OF BOUNDS and the TMA unit fills it with NaN, which the lists drop -- the
// edge days need no special path.  Cells beyond C are NaN-filled the same way (never stored).
// Two staging tiles: the copy of day i+2 is issued as soon as the four warps have read day i.
// The NaN probe is an FADD tree on the FMA pipe (a NaN, or +inf with -inf, sends the lane to the
// exact slow path), keeping the min/max pipe for the networks.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "XC_MBAR_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra XC_MBAR_DONE;\n"
      "bra XC_MBAR_WAIT;\n"
      "XC_MBAR_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

#ifndef XC_PCTL_TMA_MINBLOCKS
#define XC_PCTL_TMA_MINBLOCKS 3
#endif
#ifndef XC_PCTL_TMA_PROBE      // 0: compare chain (min/max pipe), 2: FADD tree (FMA pipe)
#define XC_PCTL_TMA_PROBE 2
#endif
constexpr int kTmaCells = kThreads;                 // cells per CTA = consumer threads
constexpr int kTmaThreads = kThreads + 32;          // + one producer warp

// values of one chunk -> descending sorted list (NaN -> -inf, counted out), cf. finish_chunk
template <int K, int NV>
__device__ __forceinline__ void finish_chunk_t(bool top, float (&v)[K], int& nv) {
#pragma unroll
  for (int k = NV; k < K; ++k) v[k] = XC_NEG_INF;
  if (!top) {
#pragma unroll
    for (int k = 0; k < NV; ++k) v[k] = -v[k];
  }
#if XC_PCTL_TMA_PROBE == 2
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < NV; ++k) acc[k & 3] = __fadd_rn(acc[k & 3], v[k]);
  const float q = __fadd_rn(__fadd_rn(acc[0], acc[1]), __fadd_rn(acc[2], acc[3]));
  const bool suspicious = (q != q);
#else
  bool suspicious = false;
#pragma unroll
  for (int k = 0; k < NV; ++k) suspicious = suspicious || (v[k] != v[k]);
#endif
  nv = NV;
  if (suspicious) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const bool bad = (v[k] != v[k]);
      nv -= bad ? 1 : 0;
      v[k] = bad ? XC_NEG_INF : v[k];
    }
  }
  if constexpr (NV == K) sort_desc<K>(v);
  else sort_desc_first<K, NV>(v);
}

template <int N2>   // years = 16 + N2, N2 in {14, 15, 16}
__global__ void __launch_bounds__(kTmaThreads, XC_PCTL_TMA_MINBLOCKS)
percentile_doy_w5t_kernel(const __grid_constant__ CUtensorMap tmap, int64_t C, int32_t L, QuantSpec spec,
                          int32_t doys_per_chunk, double* __restrict__ out, int32_t d_begin, int32_t d_end) {
  constexpr int K = 16;
  constexpr int N = K + N2;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* tile = reinterpret_cast<float*>(smem_raw);                     // [2][N][kTmaCells]
  float* sA = tile + (size_t)2 * N * kTmaCells;                         // [K][kThreads]
  float* sY = sA + (size_t)K * kThreads;                                // [2][K][kThreads]
  float* sE = sY + (size_t)2 * K * kThreads;                            // [K][kThreads]
  int* sn = reinterpret_cast<int*>(sE + (size_t)K * kThreads);          // [4][kThreads]
  uint64_t* full = reinterpret_cast<uint64_t*>(sn + 4 * kThreads);      // [2]
  uint64_t* empty = full + 2;                                           // [2]
  const int tid = threadIdx.x;
  const int p0 = d_begin + blockIdx.y * doys_per_chunk;
  const int p1 = min(d_end, p0 + doys_per_chunk);
  if (p0 >= p1) return;   // uniform over the CTA
  const int n_lists = (p1 - p0) + 4;                 // day lists e = p0-2 .. p1+1
  const int c0 = blockIdx.x * kTmaCells;
  constexpr uint32_t kTileBytes = (uint32_t)N * kTmaCells * 4u;
  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_init(&empty[0], kThreads / 32);
    mbar_init(&empty[1], kThreads / 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (tid >= kThreads) {
    // ---------------- producer warp: one elected lane issues the copies ----------------
    if (tid == kThreads) {
      for (int i = 0; i < n_lists; ++i) {
        const int st = i & 1;
        if (i >= 2) mbar_wait(&empty[st], (uint32_t)(((i >> 1) - 1) & 1));   // day i-2 has been read
        const int e = p0 - 2 + i;
        // e < 0: the day belongs to the previous year (box starts at year -1); e >= L: to the next
        const int doy = (e < 0) ? e + L : (e >= L ? e - L : e);
        const int y0 = (e < 0) ? -1 : (e >= L ? 1 : 0);
        mbar_expect_tx(&full[st], kTileBytes);
        tma_load_3d(tile + (size_t)st * N * kTmaCells, &tmap, &full[st], c0, doy, y0);
      }
    }
    return;
  }

  // ---------------- consumer warps: lane = cell ----------------
  const int lane = tid;
  const int64_t c = (int64_t)c0 + lane;
  const bool top = spec.top != 0;
  auto store_list = [&](float* dst, const float (&a)[K]) {
#pragma unroll
    for (int k = 0; k < K; ++k) dst[(size_t)k * kThreads + lane] = a[k];
  };
  float t[K], ynew[K], o[K];
  int nnew, nB = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) t[k] = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) sn[k * kThreads + lane] = 0;
  int s = 0;  // slot of Y(d-3)
#pragma unroll 1
  for (int i = 0; i < n_lists; ++i) {
    const int day = p0 - 4 + i;
    const int st = i & 1;
    {
      // Y(day + 2): the staged column -> two sorted chunks -> top-K of the day
      const float* col = tile + (size_t)st * N * kTmaCells + lane;
      float v2[K];
      mbar_wait(&full[st], (uint32_t)((i >> 1) & 1));
#pragma unroll
      for (int k = 0; k < K; ++k) ynew[k] = col[(size_t)k * kTmaCells];
#pragma unroll
      for (int k = 0; k < N2; ++k) v2[k] = col[(size_t)(K + k) * kTmaCells];
      __syncwarp();
      if ((lane & 31) == 0) mbar_arrive(&empty[st]);    // this warp has read the tile
      int n1, n2;
      finish_chunk_t<K, K>(top, ynew, n1);
      finish_chunk_t<K, N2>(top, v2, n2);
      nnew = n1 + n2;
      merge_top_desc<K>(ynew, v2);
    }
    int n;
    if ((i & 1) == 0) {
      // first day of the pair (day = d-1): ynew = Y(d+1)
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = fmaxf(sE[(size_t)k * kThreads + lane], ynew[K - 1 - k]);
      bitonic_finish_desc<K>(o);       // o <- A(d+1)
      const int nA1 = sn[3 * kThreads + lane] + nnew;
#pragma unroll
      for (int k = 0; k < K; ++k) t[k] = fmaxf(sA[(size_t)k * kThreads + lane], o[K - 1 - k]);
      bitonic_finish_desc<K>(t);       // t <- B(d)
      nB = sn[lane] + nA1;
      store_list(sA, o);
      sn[lane] = nA1;
      float* slot = sY + (size_t)s * K * kThreads;
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = slot[(size_t)k * kThreads + lane];   // Y(d-3)
      n = nB + sn[(1 + s) * kThreads + lane];
      store_list(slot, ynew);          // Y(d+1) replaces Y(d-3)
      sn[(1 + s) * kThreads + lane] = nnew;
      s ^= 1;
    } else {
      // second day of the pair (day = d): ynew = Y(d+2), the even-position list of the next pair
      store_list(sE, ynew);
      sn[3 * kThreads + lane] = nnew;
#pragma unroll
      for (int k = 0; k < K; ++k) o[k] = ynew[k];
      n = nB + nnew;
    }
    if (day < p0) continue;
    // quantile of (t U o), both sorted descending, n valid values in the window
    float u[K];
#pragma unroll
    for (int k = 0; k < K; ++k) u[k] = fmaxf(t[k], o[K - 1 - k]);
    const QuantIdx qi = quant_index(n, spec);
    const bool in_range = (n >= 2) && (qi.vi < (double)n - 1.0) && (qi.vi >= 0.0);
    const bool fast = in_range && (top ? (n - 1 - qi.ilo == K - 1) : (qi.ilo + 1 == K - 1));
    double res;
    if (__all_sync(0xffffffffu, fast)) {
      float m[K / 2];
#pragma unroll
      for (int j = 0; j < K / 2; ++j) m[j] = fminf(u[j], u[j + K / 2]);
#pragma unroll
      for (int h = K / 4; h >= 2; h >>= 1) {
#pragma unroll
        for (int j = 0; j < h; ++j) m[j] = fminf(m[j], m[j + h]);
      }
      const float smallest = fminf(m[0], m[1]), second = fmaxf(m[0], m[1]);
      res = top ? quant_lerp(smallest, second, qi) : quant_lerp(-second, -smallest, qi);
    } else {
      bitonic_finish_desc<K>(u);
      res = finalize_quantile<K>(u, n, spec);
    }
    if (c < C) out[(int64_t)day * C + c] = res;
  }
}

// ------------------------------------------------------------------------------------------------
// doy table interpolation (core/calendar.py:690-726)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
doy_interp_kernel(const double* __restrict__ tab, int32_t n_src, int64_t C, int32_t doy_min, int32_t doy_max,
                  double* __restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int n_out = doy_max - doy_min + 1;
  // source coordinates: linspace(doy_min, doy_max, n_src)
  const double step = (n_src > 1) ? ((double)(doy_max - doy_min) / (double)(n_src - 1)) : 0.0;
  for (int o = blockIdx.y; o < n_out; o += gridDim.y) {
    const double t = (double)(doy_min + o);
    // np.interp: find i with xs[i] <= t <= xs[i+1]
    int i = (step > 0.0) ? (int)floor((t - doy_min) / step) : 0;
    i = max(0, min(i, n_src - 2));
    // guard against rounding of the division: enforce xs[i] <= t < xs[i+1]
    while (i > 0 && (doy_min + i * step) > t) --i;
    while (i < n_src - 2 && (doy_min + (i + 1) * step) <= t) ++i;
    // linspace as numpy computes it: start + i*step (last point forced to stop)
    const double x0 = (i == n_src - 1) ? (double)doy_max : __dadd_rn((double)doy_min, __dmul_rn((double)i, step));
    const double x1 = (i + 1 == n_src - 1) ? (double)doy_max
                                           : __dadd_rn((double)doy_min, __dmul_rn((double)(i + 1), step));
    const double y0 = tab[(int64_t)i * C + c];
    const double y1 = tab[(int64_t)(i + 1) * C + c];
    double r;
    if (t == x1) {
      r = y1;
    } else if (t == x0) {
      r = y0;
    } else {
      // numpy's interp: slope = (y1-y0)/(x1-x0); r = slope*(t-x0) + y0
      const double slope = __ddiv_rn(__dadd_rn(y1, -y0), __dadd_rn(x1, -x0));
      r = __dadd_rn(__dmul_rn(slope, __dadd_rn(t, -x0)), y0);
    }
    out[(int64_t)o * C + c] = r;
  }
}

// ------------------------------------------------------------------------------------------------
// percentile-threshold count
// ------------------------------------------------------------------------------------------------
template <int OP, bool VALID>
__global__ void __launch_bounds__(kThreads)
doy_count_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                 const int16_t* __restrict__ doy, const double* __restrict__ table,
                 int32_t* __restrict__ out, int32_t* __restrict__ valid) {
  // blockIdx.x = period (fastest): the blocks sharing a cell range run together and share the
  // table rows through L2; blockIdx.y = cell block
  const int p = blockIdx.x;
  const int64_t c = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * 2;
  if (c >= C) return;
  const bool two = (c + 1 < C);
  const int t0 = poff[p], t1 = poff[p + 1];
  int32_t n0 = 0, n1 = 0, v0 = 0, v1 = 0;
  const float* col = x + c;
  if (two && ((ldx & 1) == 0) && ((C & 1) == 0) && ((reinterpret_cast<uintptr_t>(x) & 7u) == 0) &&
      ((reinterpret_cast<uintptr_t>(table) & 15u) == 0)) {
#pragma unroll 4
    for (int t = t0; t < t1; ++t) {
      const int d = doy[t] - 1;
      const float2 xv = *reinterpret_cast<const float2*>(col + (int64_t)t * ldx);
      const double2 th = *reinterpret_cast<const double2*>(table + (int64_t)d * C + c);
      n0 += cmpd<OP>((double)xv.x, th.x) ? 1 : 0;
      n1 += cmpd<OP>((double)xv.y, th.y) ? 1 : 0;
      if constexpr (VALID) {
        v0 += (xv.x == xv.x) ? 1 : 0;
        v1 += (xv.y == xv.y) ? 1 : 0;
      }
    }
  } else {
    for (int t = t0; t < t1; ++t) {
      const int d = doy[t] - 1;
      const float a = col[(int64_t)t * ldx];
      n0 += cmpd<OP>((double)a, table[(int64_t)d * C + c]) ? 1 : 0;
      if constexpr (VALID) v0 += (a == a) ? 1 : 0;
      if (two) {
        const float b = col[(int64_t)t * ldx + 1];
        n1 += cmpd<OP>((double)b, table[(int64_t)d * C + c + 1]) ? 1 : 0;
        if constexpr (VALID) v1 += (b == b) ? 1 : 0;
      }
    }
  }
  out[(int64_t)p * C + c] = n0;
  if (two) out[(int64_t)p * C + c + 1] = n1;
  if constexpr (VALID) {
    valid[(int64_t)p * C + c] = v0;
    if (two) valid[(int64_t)p * C + c + 1] = v1;
  }
}

// Generic periods / calendars, 4 cells per thread: the float64 table entry of (doy[t], cell) is
// folded to the float32 threshold with the same truth table (directed rounding, fold_thr) so that
// the element test is one float32 compare; 4 steps (16 B of data + 32 B of table per thread each)
// are in flight before any use.  The table rows are shared through L2 by the blocks of the same
// cell range (blockIdx.x = period is the fastest index).  Operators >, <, >=, <= only.
template <int OP, bool VALID>
__global__ void __launch_bounds__(kThreads)
doy_count4_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, const int32_t* __restrict__ poff,
                  const int16_t* __restrict__ doy, const double* __restrict__ table,
                  int32_t* __restrict__ out, int32_t* __restrict__ valid) {
  const int p = blockIdx.x;
  const int64_t c = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * 4;
  if (c >= C) return;
  const int t0 = poff[p], t1 = poff[p + 1];
  int32_t cn[4] = {0, 0, 0, 0}, vn[4] = {0, 0, 0, 0};
  const float* col = x + c;
  const double* trow = table + c;
  constexpr int U = 4;
  auto tally = [&](const float4& v, const double2& ta, const double2& tb) {
    const float thr[4] = {fold_thr<OP>(ta.x), fold_thr<OP>(ta.y), fold_thr<OP>(tb.x), fold_thr<OP>(tb.y)};
    const float xv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      cn[i] += cmp<OP>(xv[i], thr[i]) ? 1 : 0;
      if constexpr (VALID) vn[i] += (xv[i] == xv[i]) ? 1 : 0;
    }
  };
  int t = t0;
  for (; t + U <= t1; t += U) {
    float4 v[U];
    double2 ta[U], tb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int d = doy[t + u] - 1;
      v[u] = ld_stream4(col + (int64_t)(t + u) * ldx);
      ta[u] = *reinterpret_cast<const double2*>(trow + (int64_t)d * C);
      tb[u] = *reinterpret_cast<const double2*>(trow + (int64_t)d * C + 2);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) tally(v[u], ta[u], tb[u]);
  }
  for (; t < t1; ++t) {
    const int d = doy[t] - 1;
    const float4 v = ld_stream4(col + (int64_t)t * ldx);
    const double2 ta = *reinterpret_cast<const double2*>(trow + (int64_t)d * C);
    const double2 tb = *reinterpret_cast<const double2*>(trow + (int64_t)d * C + 2);
    tally(v, ta, tb);
  }
  store_vec4(out + (int64_t)p * C + c, cn);
  if constexpr (VALID) store_vec4(valid + (int64_t)p * C + c, vn);
}

// Year-blocked count for the common case "periods are whole years of equal length and the doy of a
// step is its position in the year" (noleap / 360_day, freq YS): a thread owns 4 adjacent cells and
// YB consecutive years, so every table row is fetched once per YB years instead of once per year
// (the table is 365*C*8 B = 3 GB at full size, far beyond L2), and it is folded once per row into a
// float32 threshold by directed rounding (x op t64  <=>  x op' t32 for every float32 x), which turns
// the per-element float64 compare + conversion into one float32 compare.
template <int OP, int YB, bool VALID>
__global__ void __launch_bounds__(kThreads)
doy_count_years_kernel(const float* __restrict__ x, int64_t C, int64_t ldx, int64_t first_row, int32_t n_years,
                       int32_t L, const double* __restrict__ table, int32_t* __restrict__ out,
                       int32_t* __restrict__ valid) {
  // blockIdx.x = year group (fastest: groups of one cell range run together and share table rows in L2)
  const int y0 = blockIdx.x * YB;
  const int64_t c = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * 4;
  if (c >= C) return;
  // packed counters: low 16 bits = exceedance count, high 16 bits = valid count (both <= 366)
  uint32_t acc[YB][4];
#pragma unroll
  for (int j = 0; j < YB; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[j][i] = 0u;
  const int ny = min(YB, n_years - y0);
  const float* base = x + (first_row + (int64_t)y0 * L) * ldx + c;
  const int64_t ystride = (int64_t)L * ldx;
  const double* trow = table + c;
  auto row = [&](int d, double2& ta, double2& tb, float4 (&v)[YB]) {
    ta = *reinterpret_cast<const double2*>(trow + (int64_t)d * C);
    tb = *reinterpret_cast<const double2*>(trow + (int64_t)d * C + 2);
#pragma unroll
    for (int j = 0; j < YB; ++j)
      if (j < ny) v[j] = ld_stream4(base + (int64_t)j * ystride + (int64_t)d * ldx);
  };
  auto tally = [&](const double2& ta, const double2& tb, const float4 (&v)[YB]) {
    const float thr[4] = {fold_thr<OP>(ta.x), fold_thr<OP>(ta.y), fold_thr<OP>(tb.x), fold_thr<OP>(tb.y)};
#pragma unroll
    for (int j = 0; j < YB; ++j) {
      if (j < ny) {
        const float xv[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[j][i] += cmp<OP>(xv[i], thr[i]) ? 1u : 0u;
          if constexpr (VALID) acc[j][i] += (xv[i] == xv[i]) ? 65536u : 0u;
        }
      }
    }
  };
  int d = 0;
  for (; d + 2 <= L; d += 2) {  // two table rows and 2*YB data rows in flight before any use
    double2 ta0, tb0, ta1, tb1;
    float4 v0[YB], v1[YB];
    row(d, ta0, tb0, v0);
    row(d + 1, ta1, tb1, v1);
    tally(ta0, tb0, v0);
    tally(ta1, tb1, v1);
  }
  for (; d < L; ++d) {
    double2 ta, tb;
    float4 v[YB];
    row(d, ta, tb, v);
    tally(ta, tb, v);
  }
#pragma unroll
  for (int j = 0; j < YB; ++j) {
    if (j < ny) {
      const int32_t cn[4] = {(int32_t)(acc[j][0] & 0xffffu), (int32_t)(acc[j][1] & 0xffffu),
                             (int32_t)(acc[j][2] & 0xffffu), (int32_t)(acc[j][3] & 0xffffu)};
      store_vec4(out + (int64_t)(y0 + j) * C + c, cn);
      if constexpr (VALID) {
        const int32_t vn[4] = {(int32_t)(acc[j][0] >> 16), (int32_t)(acc[j][1] >> 16), (int32_t)(acc[j][2] >> 16),
                               (int32_t)(acc[j][3] >> 16)};
        store_vec4(valid + (int64_t)(y0 + j) * C + c, vn);
      }
    }
  }
}

template <int K>
int32_t launch_generic(const float* x, int64_t T, int64_t C, int64_t ldx, const int32_t* pos, int32_t n_doy,
                       int32_t n_years, int32_t h, const QuantSpec& spec, double* out, cudaStream_t st,
                       int d_begin = 0, int d_end = -1, const int32_t* vrow = nullptr) {
  if (d_end < 0) d_end = n_doy;
  const int nd = d_end - d_begin;
  if (nd <= 0) return XC_OK;
  const int64_t cblocks = (C + kThreads - 1) / kThreads;
  // enough chunks to fill the machine when the grid is narrow
  int chunks = (int)((sm_count() * 8 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : (chunks > nd ? nd : chunks);
  const int per = (nd + chunks - 1) / chunks;
  chunks = (nd + per - 1) / per;
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  percentile_doy_generic_kernel<K><<<grid, kThreads, 0, st>>>(x, T, C, ldx, pos, n_doy, n_years, h, spec, per, out,
                                                              d_begin, d_end, vrow);
  return launch_status("percentile_doy_generic_kernel");
}

// pos == nullptr: uniform years (days [0, L)); else table mode on the interior days [d_begin, d_end)
template <int K>
int32_t launch_uniform(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t L, int32_t N, int32_t W,
                       const QuantSpec& spec, double* out, cudaStream_t st, const int32_t* pos = nullptr,
                       int n_doy = 0, int d_begin = 0, int d_end = -1) {
  if (d_end < 0) d_end = L;
  const int nd = d_end - d_begin;
  if (nd <= 0) return XC_OK;
  const int64_t cblocks = (C + kThreads - 1) / kThreads;
  int chunks = (int)((sm_count() * 12 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : chunks;
  int per = (nd + chunks - 1) / chunks;
  if (per < 8 * W) per = 8 * W;  // keep the halo overhead (W-1 extra day lists per chunk) small
  if (per > nd) per = nd;
  chunks = (nd + per - 1) / per;
  const size_t smem = (size_t)(W - 1) * (K + 1) * kThreads * 4;
  if (smem > 48 * 1024) {
    cudaError_t e = pos ? cudaFuncSetAttribute(percentile_doy_uniform_kernel<K, true>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                        : cudaFuncSetAttribute(percentile_doy_uniform_kernel<K, false>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(percentile_doy_uniform_kernel)");
  }
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  if (pos)
    percentile_doy_uniform_kernel<K, true><<<grid, kThreads, smem, st>>>(x, (int32_t)T, C, ldx, L, N, W, spec, per,
                                                                         out, pos, n_doy, d_begin, d_end);
  else
    percentile_doy_uniform_kernel<K, false><<<grid, kThreads, smem, st>>>(x, (int32_t)T, C, ldx, L, N, W, spec, per,
                                                                          out, pos, n_doy, d_begin, d_end);
  return launch_status("percentile_doy_uniform_kernel");
}

template <int K>
int32_t launch_w5(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t L, int32_t N, const QuantSpec& spec,
                  double* out, cudaStream_t st, const int32_t* pos = nullptr, int n_doy = 0, int d_begin = 0,
                  int d_end = -1) {
  if (d_end < 0) d_end = L;
  const int nd = d_end - d_begin;
  if (nd <= 0) return XC_OK;
  const int64_t cblocks = (C + kThreads - 1) / kThreads;
  int chunks = (int)((sm_count() * 16 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : chunks;
  int per = (nd + chunks - 1) / chunks;
  if (per < 40) per = 40;  // 4 extra day lists per chunk
  per = (per + 1) & ~1;    // whole pairs of days
  if (per > nd) per = nd;
  chunks = (nd + per - 1) / per;
  // 4 lists + 4 counts per lane, plus the 32-row staging column of the cp.async prefetch
  const size_t smem = (size_t)4 * (K + 1) * kThreads * 4 + (XC_PCTL_STAGE && K == 16 && !pos ? (size_t)32 * kThreads * 4 : 0);
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  if (smem > 48 * 1024) {
    cudaError_t e = pos ? cudaFuncSetAttribute(percentile_doy_w5p_kernel<K, true>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                        : cudaFuncSetAttribute(percentile_doy_w5p_kernel<K, false>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(percentile_doy_w5p_kernel)");
  }
  if (pos)
    percentile_doy_w5p_kernel<K, true><<<grid, kThreads, smem, st>>>(x, (int32_t)T, C, ldx, L, N, spec, per, out, pos,
                                                                     n_doy, d_begin, d_end);
  else
    percentile_doy_w5p_kernel<K, false><<<grid, kThreads, smem, st>>>(x, (int32_t)T, C, ldx, L, N, spec, per, out,
                                                                      pos, n_doy, d_begin, d_end);
  return launch_status("percentile_doy_w5p_kernel");
}


// TMA path of launch_w5<16>: needs a 16-byte aligned base, ldx % 4 == 0 (global strides are multiples of
// 16 bytes) and 30..32 years.  Returns 1 when the shape does not qualify (caller falls back).
typedef CUresult (*XcEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static XcEncodeTiled tensor_map_encoder() {
  static XcEncodeTiled fn = []() -> XcEncodeTiled {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess) {
      (void)cudaGetLastError();
      return nullptr;
    }
    return (XcEncodeTiled)p;
  }();
  return fn;
}

int32_t launch_w5_tma(const float* x, int64_t T, int64_t C, int64_t ldx, int32_t L, int32_t N, const QuantSpec& spec,
                      double* out, cudaStream_t st) {
  if (N < 30 || N > 32 || (ldx % 4) != 0 || !aligned16(x) || T != (int64_t)L * N || L < 8) return 1;
  if (C > 2147483647LL - kTmaCells) return 1;
  XcEncodeTiled enc = tensor_map_encoder();
  if (!enc) return 1;
  CUtensorMap map;
  const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)L, (cuuint64_t)N};
  const cuuint64_t strides[2] = {(cuuint64_t)ldx * 4ull, (cuuint64_t)L * (cuuint64_t)ldx * 4ull};
  const cuuint32_t box[3] = {(cuuint32_t)kTmaCells, 1u, (cuuint32_t)N};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(x), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NAN_REQUEST_ZERO_FMA);
  if (r != CUDA_SUCCESS) return 1;
  const int nd = L;
  const int64_t cblocks = (C + kTmaCells - 1) / kTmaCells;
  int chunks = (int)((sm_count() * 12 + cblocks - 1) / cblocks);
  chunks = chunks < 1 ? 1 : chunks;
  int per = (nd + chunks - 1) / chunks;
  if (per < 40) per = 40;  // 4 extra day lists per chunk
  per = (per + 1) & ~1;    // whole pairs of days
  if (per > nd) per = nd;
  chunks = (nd + per - 1) / per;
  const size_t smem = (size_t)2 * N * kTmaCells * 4 + (size_t)4 * (16 + 1) * kThreads * 4 + 64;
  dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
  auto go = [&](auto kern) -> int32_t {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_fail(e, "cudaFuncSetAttribute(percentile_doy_w5t_kernel)");
    kern<<<grid, kTmaThreads, smem, st>>>(map, C, L, spec, per, out, 0, L);
    return launch_status("percentile_doy_w5t_kernel");
  };
  if (N == 30) return go(percentile_doy_w5t_kernel<14>);
  if (N == 31) return go(percentile_doy_w5t_kernel<15>);
  return go(percentile_doy_w5t_kernel<16>);
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int64_t xc_percentile_doy_workspace_bytes(int64_t T, int64_t C, int32_t n_doy, int32_t n_years,
                                                     int32_t window, int32_t n_per) {
  (void)C; (void)window; (void)n_per;
  // (year, doy) -> step table, the same table through the virtual-row map, and the map itself
  return 2 * (int64_t)n_doy * (int64_t)n_years * 4 + T * 4 + 256;
}

static int32_t percentile_doy_impl(const float* x, int64_t T, int64_t C, int64_t ldx,
                                   const int16_t* doy_index_host, const int16_t* year_index_host,
                                   int32_t n_doy, int32_t n_years, int32_t window,
                                   const double* percentiles_host, int32_t n_per, double alpha, double beta,
                                   double* out, void* workspace, int64_t workspace_bytes, void* stream,
                                   const int32_t* vrow_host) {
  XC_REQUIRE(x && doy_index_host && year_index_host && percentiles_host && out, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && T < 2147483647LL, "bad shape");
  XC_REQUIRE(n_doy > 0 && n_doy <= 366 && n_years > 0 && n_per > 0, "bad calendar description");
  XC_REQUIRE(window >= 1, "window must be >= 1");
  if (window % 2 == 0) {
    set_error("even `window` (xarray's center=True convention for even windows) is not supported");
    return XC_ERR_UNSUPPORTED;
  }
  const int h = window / 2;
  cudaStream_t st = (cudaStream_t)stream;

  // (year, doy) -> row table, and detection of the uniform-year fast path
  std::vector<int32_t> pos((size_t)n_doy * n_years, -1);
  bool uniform = (T == (int64_t)n_doy * n_years);
  for (int64_t t = 0; t < T; ++t) {
    const int d = doy_index_host[t], y = year_index_host[t];
    XC_REQUIRE(d >= 1 && d <= n_doy && y >= 0 && y < n_years, "doy/year index out of range at step %lld", (long long)t);
    pos[(size_t)y * n_doy + (d - 1)] = (int32_t)t;
    if (uniform && (d - 1 != (int)(t % n_doy) || y != (int)(t / n_doy))) uniform = false;
  }
  int32_t* pos_d = nullptr;      // (year, doy) -> step
  int32_t* posrow_d = nullptr;   // (year, doy) -> row holding that step's value (== pos_d without vrow)
  int32_t* vrow_d = nullptr;     // step -> row
  if (vrow_host) uniform = false;
  if (!uniform) {
    const int64_t nb = (int64_t)pos.size() * 4;
    const int64_t need = vrow_host ? 2 * nb + T * 4 : nb;
    XC_REQUIRE(workspace != nullptr && workspace_bytes >= need, "workspace too small: need %lld bytes", (long long)need);
    pos_d = (int32_t*)workspace;
    posrow_d = pos_d;
    XC_CHECK_CUDA(cudaMemcpyAsync(pos_d, pos.data(), (size_t)nb, cudaMemcpyHostToDevice, st));
    std::vector<int32_t> posrow;
    if (vrow_host) {
      for (int64_t t = 0; t < T; ++t)
        XC_REQUIRE(vrow_host[t] >= -1 && vrow_host[t] < T, "virtual row out of range at step %lld", (long long)t);
      posrow.resize(pos.size());
      for (size_t k = 0; k < pos.size(); ++k) posrow[k] = pos[k] < 0 ? -1 : vrow_host[pos[k]];
      posrow_d = pos_d + pos.size();
      vrow_d = posrow_d + pos.size();
      XC_CHECK_CUDA(cudaMemcpyAsync(posrow_d, posrow.data(), (size_t)nb, cudaMemcpyHostToDevice, st));
      XC_CHECK_CUDA(cudaMemcpyAsync(vrow_d, vrow_host, (size_t)T * 4, cudaMemcpyHostToDevice, st));
    }
    // the tables live on this stack frame: make sure the copies have been issued from pageable memory
    XC_CHECK_CUDA(cudaStreamSynchronize(st));
  }

  // interior days whose windows never leave the year: [h, L_int - h) with L_int the shortest full year
  const int L_int = (n_doy == 366) ? 365 : n_doy;
  for (int ip = 0; ip < n_per; ++ip) {
    const double per = percentiles_host[ip];
    XC_REQUIRE(per >= 0.0 && per <= 100.0, "percentiles must be in [0, 100], got %g", per);
    QuantSpec spec;
    const int need = plan_quantile(per, alpha, beta, n_years * window, &spec);
    if (need < 0) {
      set_error("percentile %g with alpha=%g beta=%g: plotting positions outside [0, 1] are not supported", per,
                alpha, beta);
      return XC_ERR_UNSUPPORTED;
    }
    double* o = out + (int64_t)ip * n_doy * C;
    if (need > 64) {
      // order statistics far from both ends of the sample (e.g. the median): selection kernel
      const int nmax = n_years * window;
      if (nmax > 768) {
        set_error("percentile %g of up to %d samples: the selection kernel holds at most 768 samples per cell", per,
                  nmax);
        return XC_ERR_UNSUPPORTED;
      }
      if (pos_d == nullptr) {
        const int64_t nbytes = (int64_t)pos.size() * 4;
        XC_REQUIRE(workspace != nullptr && workspace_bytes >= nbytes, "workspace too small: need %lld bytes",
                   (long long)nbytes);
        pos_d = (int32_t*)workspace;
        posrow_d = pos_d;
        XC_CHECK_CUDA(cudaMemcpyAsync(pos_d, pos.data(), (size_t)nbytes, cudaMemcpyHostToDevice, st));
        XC_CHECK_CUDA(cudaStreamSynchronize(st));
      }
      const size_t smem = (size_t)nmax * kSelThreads * 4;
      if (smem > 48 * 1024)
        XC_CHECK_CUDA(cudaFuncSetAttribute(percentile_doy_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)smem));
      const int64_t cblocks = (C + kSelThreads - 1) / kSelThreads;
      int chunks = (int)((sm_count() * 8 + cblocks - 1) / cblocks);
      chunks = chunks < 1 ? 1 : (chunks > n_doy ? n_doy : chunks);
      const int per_chunk = (n_doy + chunks - 1) / chunks;
      chunks = (n_doy + per_chunk - 1) / per_chunk;
      dim3 grid((unsigned)cblocks, (unsigned)chunks, 1);
      percentile_doy_select_kernel<<<grid, kSelThreads, smem, st>>>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec,
                                                                    per_chunk, o, vrow_d);
      const int32_t es = launch_status("percentile_doy_select_kernel");
      if (es) return es;
      continue;
    }
    const int kk = need <= 8 ? 8 : need <= 16 ? 16 : 32;
    const size_t smem_need = (size_t)(window - 1) * (kk + 1) * kThreads * 4;
    const bool fast_ok = window >= 3 && need <= 32 && smem_need <= 200 * 1024 && (L_int - 2 * h) >= 8;
    int32_t e = XC_OK;
    if (uniform && fast_ok) {
      if (window == 5 && need <= 16) {
        e = 1;
        if (need > 8 && !getenv("XCLIM_B200_NO_TMA")) e = launch_w5_tma(x, T, C, ldx, n_doy, n_years, spec, o, st);
        if (e == 1)
          e = need <= 8 ? launch_w5<8>(x, T, C, ldx, n_doy, n_years, spec, o, st)
                        : launch_w5<16>(x, T, C, ldx, n_doy, n_years, spec, o, st);
      } else
        e = need <= 8    ? launch_uniform<8>(x, T, C, ldx, n_doy, n_years, window, spec, o, st)
            : need <= 16 ? launch_uniform<16>(x, T, C, ldx, n_doy, n_years, window, spec, o, st)
                         : launch_uniform<32>(x, T, C, ldx, n_doy, n_years, window, spec, o, st);
    } else {
      if (pos_d == nullptr) {  // uniform calendar without a fast instantiation: the table is still needed
        const int64_t nbytes = (int64_t)pos.size() * 4;
        XC_REQUIRE(workspace != nullptr && workspace_bytes >= nbytes, "workspace too small: need %lld bytes",
                   (long long)nbytes);
        pos_d = (int32_t*)workspace;
        posrow_d = pos_d;
        XC_CHECK_CUDA(cudaMemcpyAsync(pos_d, pos.data(), (size_t)nbytes, cudaMemcpyHostToDevice, st));
        XC_CHECK_CUDA(cudaStreamSynchronize(st));
      }
      // Days whose samples decompose into per-day lists: the window must stay inside the year
      // ([h, L_int - h)) and no window centre may fall outside the series (the h days before the first
      // step's day-of-year and after the last step's: their neighbours exist but their centres do not).
      std::vector<char> fast_day((size_t)n_doy, 0);
      if (fast_ok) {
        for (int d = h; d < L_int - h; ++d) fast_day[d] = 1;
        const int s0 = doy_index_host[0] - 1, e1 = doy_index_host[T - 1] - 1;
        for (int d = s0 - h; d < s0; ++d)
          if (d >= 0) fast_day[d] = 0;
        for (int d = e1 + 1; d <= e1 + h; ++d)
          if (d < n_doy) fast_day[d] = 0;
      }
      for (int a = 0; a < n_doy;) {
        int b = a;
        const bool fast = fast_day[a] != 0;
        while (b < n_doy && (fast_day[b] != 0) == fast) ++b;
        if (fast && (b - a) >= 8) {
          if (window == 5 && need <= 16)
            e = need <= 8 ? launch_w5<8>(x, T, C, ldx, n_doy, n_years, spec, o, st, posrow_d, n_doy, a, b)
                          : launch_w5<16>(x, T, C, ldx, n_doy, n_years, spec, o, st, posrow_d, n_doy, a, b);
          else
            e = need <= 8    ? launch_uniform<8>(x, T, C, ldx, n_doy, n_years, window, spec, o, st, posrow_d, n_doy, a, b)
                : need <= 16 ? launch_uniform<16>(x, T, C, ldx, n_doy, n_years, window, spec, o, st, posrow_d, n_doy, a, b)
                             : launch_uniform<32>(x, T, C, ldx, n_doy, n_years, window, spec, o, st, posrow_d, n_doy,
                                                  a, b);
        } else {
          if (need <= 4) e = launch_generic<4>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, o, st, a, b, vrow_d);
          else if (need <= 8) e = launch_generic<8>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, o, st, a, b, vrow_d);
          else if (need <= 16) e = launch_generic<16>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, o, st, a, b, vrow_d);
          else if (need <= 32) e = launch_generic<32>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, o, st, a, b, vrow_d);
          else e = launch_generic<64>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, o, st, a, b, vrow_d);
        }
        if (e) return e;
        a = b;
      }
    }
    if (e) return e;
  }
  return XC_OK;
}

extern "C" int32_t xc_percentile_doy_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                         const int16_t* doy_index_host, const int16_t* year_index_host,
                                         int32_t n_doy, int32_t n_years, int32_t window,
                                         const double* percentiles_host, int32_t n_per, double alpha, double beta,
                                         double* out, void* workspace, int64_t workspace_bytes, void* stream) {
  return percentile_doy_impl(x, T, C, ldx, doy_index_host, year_index_host, n_doy, n_years, window,
                             percentiles_host, n_per, alpha, beta, out, workspace, workspace_bytes, stream, nullptr);
}

extern "C" int32_t xc_percentile_doy_vrow_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                              const int16_t* doy_index_host, const int16_t* year_index_host,
                                              const int32_t* vrow_host, int32_t n_doy, int32_t n_years,
                                              int32_t window, const double* percentiles_host, int32_t n_per,
                                              double alpha, double beta, double* out, void* workspace,
                                              int64_t workspace_bytes, void* stream) {
  XC_REQUIRE(vrow_host != nullptr, "null pointer argument");
  return percentile_doy_impl(x, T, C, ldx, doy_index_host, year_index_host, n_doy, n_years, window,
                             percentiles_host, n_per, alpha, beta, out, workspace, workspace_bytes, stream, vrow_host);
}

// Forces the generic kernel (test hook: the two paths must agree bit for bit).
extern "C" int32_t xc_percentile_doy_generic_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                                 const int16_t* doy_index_host, const int16_t* year_index_host,
                                                 int32_t n_doy, int32_t n_years, int32_t window, double percentile,
                                                 double alpha, double beta, double* out, void* workspace,
                                                 int64_t workspace_bytes, void* stream) {
  XC_REQUIRE(x && doy_index_host && year_index_host && out && workspace, "null pointer argument");
  XC_REQUIRE(window >= 1 && window % 2 == 1, "window must be odd");
  std::vector<int32_t> pos((size_t)n_doy * n_years, -1);
  for (int64_t t = 0; t < T; ++t) {
    const int d = doy_index_host[t], y = year_index_host[t];
    XC_REQUIRE(d >= 1 && d <= n_doy && y >= 0 && y < n_years, "doy/year index out of range");
    pos[(size_t)y * n_doy + (d - 1)] = (int32_t)t;
  }
  const int64_t need_b = (int64_t)pos.size() * 4;
  XC_REQUIRE(workspace_bytes >= need_b, "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  XC_CHECK_CUDA(cudaMemcpyAsync(workspace, pos.data(), (size_t)need_b, cudaMemcpyHostToDevice, st));
  XC_CHECK_CUDA(cudaStreamSynchronize(st));
  QuantSpec spec;
  const int need = plan_quantile(percentile, alpha, beta, n_years * window, &spec);
  if (need < 0 || need > 64) {
    set_error("percentile needs %d order statistics; at most 64 are kept", need);
    return XC_ERR_UNSUPPORTED;
  }
  const int32_t* pos_d = (const int32_t*)workspace;
  const int h = window / 2;
  if (need <= 4) return launch_generic<4>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, out, st);
  if (need <= 8) return launch_generic<8>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, out, st);
  if (need <= 16) return launch_generic<16>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, out, st);
  if (need <= 32) return launch_generic<32>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, out, st);
  return launch_generic<64>(x, T, C, ldx, pos_d, n_doy, n_years, h, spec, out, st);
}

extern "C" int32_t xc_doy_interp_f64(const double* table, int32_t n_src, int64_t C, int32_t doy_min,
                                     int32_t doy_max, double* out, void* stream) {
  XC_REQUIRE(table && out, "null pointer argument");
  XC_REQUIRE(n_src >= 2 && C > 0 && doy_max > doy_min, "bad shape");
  const int n_out = doy_max - doy_min + 1;
  dim3 grid((unsigned)((C + 255) / 256), (unsigned)(n_out < 64 ? n_out : 64), 1);
  doy_interp_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(table, n_src, C, doy_min, doy_max, out);
  return launch_status("doy_interp_kernel");
}

extern "C" int32_t xc_doy_threshold_count_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                              const int32_t* period_offsets, int32_t P,
                                              const int16_t* doy_index, const double* table, int32_t n_doy,
                                              int32_t op, int32_t* out_count, int32_t* valid_count, void* stream) {
  XC_REQUIRE(x && period_offsets && doy_index && table && out_count, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && P > 0 && n_doy > 0, "bad shape");
  (void)n_doy;
  cudaStream_t st = (cudaStream_t)stream;
  // 4 cells per thread with float32-folded thresholds when the layout allows 128-bit accesses and the
  // operator is an inequality
  const bool vec4 = (C % 4 == 0) && (ldx % 4 == 0) && aligned16(x) && aligned16(table) && aligned16(out_count) &&
                    (valid_count == nullptr || aligned16(valid_count)) && op >= XC_OP_GT && op <= XC_OP_LE;
  if (vec4) {
    const int64_t cb4 = (C / 4 + kThreads - 1) / kThreads;
    XC_REQUIRE(cb4 <= 65535, "too many cells for one launch: tile the grid by latitude");
    dim3 grid4((unsigned)P, (unsigned)cb4, 1);
    return dispatch_op(op, [&](auto OPC) -> int32_t {
      constexpr int OP = decltype(OPC)::value;
      if constexpr (OP == XC_OP_EQ || OP == XC_OP_NE) {
        return XC_ERR_INVALID;  // unreachable: vec4 requires an inequality
      } else {
        if (valid_count)
          doy_count4_kernel<OP, true><<<grid4, kThreads, 0, st>>>(x, C, ldx, period_offsets, doy_index, table,
                                                                  out_count, valid_count);
        else
          doy_count4_kernel<OP, false><<<grid4, kThreads, 0, st>>>(x, C, ldx, period_offsets, doy_index, table,
                                                                   out_count, valid_count);
        return launch_status("doy_count4_kernel");
      }
    });
  }
  const int64_t pairs = (C + 1) / 2;
  const int64_t cblocks = (pairs + kThreads - 1) / kThreads;
  XC_REQUIRE(cblocks <= 65535, "too many cells for one launch: tile the grid by latitude");
  dim3 grid((unsigned)P, (unsigned)cblocks, 1);
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    if (valid_count)
      doy_count_kernel<OP, true><<<grid, kThreads, 0, st>>>(x, C, ldx, period_offsets, doy_index, table, out_count,
                                                            valid_count);
    else
      doy_count_kernel<OP, false><<<grid, kThreads, 0, st>>>(x, C, ldx, period_offsets, doy_index, table, out_count,
                                                             valid_count);
    return launch_status("doy_count_kernel");
  });
}

extern "C" int32_t xc_doy_threshold_count_years_f32(const float* x, int64_t T, int64_t C, int64_t ldx,
                                                    int64_t first_row, int32_t n_years, int32_t year_len,
                                                    const double* table, int32_t op, int32_t* out_count,
                                                    int32_t* valid_count, void* stream) {
  XC_REQUIRE(x && table && out_count, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C && n_years > 0 && year_len > 0, "bad shape");
  XC_REQUIRE(first_row >= 0 && first_row + (int64_t)n_years * year_len <= T, "years outside the series");
  XC_REQUIRE(op >= XC_OP_GT && op <= XC_OP_LE, "Operation `%d` not permitted for indice.", op);
  XC_REQUIRE((C % 4 == 0) && (ldx % 4 == 0) && aligned16(x) && aligned16(table) && aligned16(out_count) &&
                 (valid_count == nullptr || aligned16(valid_count)),
             "xc_doy_threshold_count_years_f32 needs C, ldx multiples of 4 and 16-byte aligned buffers");
  constexpr int YB = 3;
  XC_REQUIRE(year_len <= 65535, "year length too large for the packed counters");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cblocks = (C / 4 + kThreads - 1) / kThreads;
  XC_REQUIRE(cblocks <= 65535, "too many cells for one launch: tile the grid by latitude");
  dim3 grid((unsigned)((n_years + YB - 1) / YB), (unsigned)cblocks, 1);
  return dispatch_op(op, [&](auto OPC) -> int32_t {
    constexpr int OP = decltype(OPC)::value;
    if constexpr (OP <= XC_OP_LE) {
      if (valid_count)
        doy_count_years_kernel<OP, YB, true><<<grid, kThreads, 0, st>>>(x, C, ldx, first_row, n_years, year_len, table,
                                                                        out_count, valid_count);
      else
        doy_count_years_kernel<OP, YB, false><<<grid, kThreads, 0, st>>>(x, C, ldx, first_row, n_years, year_len,
                                                                         table, out_count, valid_count);
    }
    return launch_status("doy_count_years_kernel");
  });
}
