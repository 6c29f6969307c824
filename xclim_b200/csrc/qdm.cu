// Quantile delta mapping (sdba / xsdba `QuantileDeltaMapping`, group="time"): the adjust step.
//
// The arithmetic lives in the third-party package xsdba (re-exported by sdba.py:11) whose sources are NOT under
// /root/reference: this file restates the published algorithm (PARITY UNPINNED, see DESIGN.md).  Its train step
// is EmpiricalQuantileMapping.train unchanged (eqm.cu); adjust, per cell of sim:
//   rank   : r = average 1-based rank of x among the n valid values of the cell's whole series
//            (bottleneck.nanrankdata), p = r / n (xarray rank(pct=True)), sim_q = (mx * (p - mn)) / (mx - mn)
//            with mn, mx the min, max of p over the cell (xsdba.utils.rank, reference CHANGELOG.rst:1043); float64.
//   factor : scipy interp1d(nodes, af, kind=interp, bounds_error=False, fill_value=(first, last valid af)) at
//            sim_q, the NaN entries of af dropped, cast to float32 (xsdba's _interp_on_quantiles_1D); linear
//            evaluates the two-weight form of scipy's interp1d._call_linear (its float32 node differences included).
//   correct: scen = sim + af_t ("+") or sim * af_t ("*") in float32.
//
// Design.  The rank is a statistic of the whole series of a cell, and in the (time, cell) layout that series sits
// at a 4 MB row stride: what costs is the number of (CTA, time row) touches, whatever the bytes per touch (see
// the EQM train notes in eqm.cu).  So no kernel walks one cell down the rows:
//   (1) qdm_transpose_kernel copies a chunk of cells to cell-major scratch through 32 x 32 shared-memory tiles
//       (128-byte touches: T * C / 32 of them);
//   (2) qdm_rank_kernel, one CTA per cell, reads its contiguous series (4 sweeps, the first from HBM, the others
//       mostly from L2), counting-sorts it into 1 + K + 1 monotone value bins (-inf | the finite range | +inf,
//       K = NPAD / 4), and ranks every element as (elements of the lower bins) + (elements of its own bin below
//       it / equal to it).  Bins that hold one value (dry days, quantised data, infinities) cost nothing; the
//       others are compared element by element.  A cell where that would exceed 32 comparisons per element (a
//       range stretched by outliers, +-3e38 next to ordinary values) sorts its valid values instead (bitonic
//       sort in shared memory) and ranks by binary search: the same ranks.  It writes the doubled rank
//       2r - 2 as a uint16 (0xffff = NaN) per element and (n, min, max code) per cell;
//   (3) qdm_apply_kernel streams sim in (time, cell) order, takes the ranks through a 32 x 32 transposing tile,
//       rescales in float64, interpolates against the cell's compacted (valid af) node table -- a computed
//       index from the nearly uniform nodes plus exact steps replaces the search -- and writes scen (and
//       sim_q).
// HBM traffic per element: sim 4 + scratch 4 (write) + 4 (read) + ranks 2 + 2 + sim 4 + scen 4 = 24 bytes,
// plus 8 for sim_q (algorithmic: 8, plus 8).  Scratch is 6 T + 16 bytes per cell; the entry point walks the cells
// in chunks that fit the workspace it is given.
// Measured on an H100 80GB HBM3 (SXM, 400 W power limit), T = 10950, 180 x 1440 cells, nq = 20, linear, 2 GiB of
// scratch (8 chunks): 87 ms per adjust (rank 38.8 ms, apply 33.9 ms, transpose 13.3 ms), 93 ms with sim_q (apply
// 37.3 ms).  No other design was built or measured.
#include <float.h>
#include <limits.h>

#include <algorithm>

#include "qmap.cuh"

namespace xc {
namespace {

constexpr int kTile = 32;                // transposing tiles: 32 cells x 32 steps, 32 x 8 threads
constexpr int kRankThreads = 512;
constexpr int kRankWarps = kRankThreads / 32;
constexpr int kCountBudget = 32;         // in-bin comparisons per element above which the cell is sorted instead
constexpr unsigned kNanRank = 0xffffu;   // rank code of a NaN element
constexpr int64_t kMaxSteps = 32768;     // uint16 rank codes: 2 n - 1 <= 65535

__host__ __device__ inline int64_t align16(int64_t b) { return (b + 15) & ~(int64_t)15; }

// scratch of one chunk of nc cells: cell-major values | rank codes | per-cell stats
inline int64_t chunk_bytes(int64_t T, int64_t nc) { return align16(nc * T * 4) + align16(nc * T * 2) + nc * 16; }

// (1) sim columns [0, nc) (time, cell) -> xt (cell, time)
__global__ void __launch_bounds__(kTile * 8)
qdm_transpose_kernel(const float* __restrict__ sim, int64_t T, int64_t ldx, int64_t nc, float* __restrict__ xt) {
  __shared__ float tile[kTile][kTile + 1];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t cb = (int64_t)blockIdx.x * kTile, tb = (int64_t)blockIdx.y * kTile;
  for (int k = ty; k < kTile; k += 8) {
    const int64_t t = tb + k, c = cb + tx;
    if (t < T && c < nc) tile[k][tx] = ld_stream(sim + t * ldx + c);
  }
  __syncthreads();
  for (int k = ty; k < kTile; k += 8) {
    const int64_t c = cb + k, t = tb + tx;
    if (t < T && c < nc) xt[c * T + t] = tile[tx][k];
  }
}

// all threads of the CTA get op over the CTA; red: kRankWarps slots
template <typename V, typename Op>
__device__ __forceinline__ V block_reduce(V v, Op op, V* red) {
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();  // the previous reduction through `red` is read by every thread
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < kRankWarps; ++w) v = op(v, red[w]);
  return v;
}

// in-place exclusive prefix sum of a[0 .. K) by the CTA (consecutive runs of K / kRankThreads per thread)
template <int K>
__device__ __forceinline__ void block_exclusive_scan(int* a, int* red) {
  constexpr int per = (K + kRankThreads - 1) / kRankThreads;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int i0 = tid * per;
  int loc[per], sum = 0;
#pragma unroll
  for (int i = 0; i < per; ++i) {
    loc[i] = (i0 + i < K) ? a[i0 + i] : 0;
    sum += loc[i];
  }
  int incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const int up = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += up;
  }
  if (lane == 31) red[wid] = incl;
  __syncthreads();
  int run = incl - sum;
  for (int w = 0; w < wid; ++w) run += red[w];
#pragma unroll
  for (int i = 0; i < per; ++i) {
    if (i0 + i < K) a[i0 + i] = run;
    run += loc[i];
  }
}

// value bin: -inf -> 0, finite -> 1 .. K - 2 by a monotone affine map of the finite range, +inf -> K - 1.  Any
// monotone binning gives the same ranks; this one keeps the bins of ordinary data small.
template <int K>
__device__ __forceinline__ int bin_of(float v, float s, float o) {
  if (v == -INFINITY) return 0;
  if (v == INFINITY) return K - 1;
  return 1 + min(max(__float2int_rz(fmaf(v, s, o)), 0), K - 3);
}

__device__ __forceinline__ int lower_bound(const float* keys, int n, float v) {   // first i with keys[i] >= v
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ int upper_bound(const float* keys, int n, float v) {   // first i with keys[i] > v
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// (2) one CTA per cell: rank codes 2 r - 2 of the cell's series xt[c * T ..] (T <= NPAD), stats (n, min code, max
// code).  Shared memory: values grouped by bin [T] | bin ends [K] | one-value flags [K / 32]; the fallback sort
// reuses it as NPAD keys.
template <int NPAD>
__global__ void __launch_bounds__(kRankThreads)
qdm_rank_kernel(const float* __restrict__ xt, int32_t T, uint16_t* __restrict__ rk, int4* __restrict__ stats) {
  constexpr int K = NPAD / 4;
  extern __shared__ __align__(16) unsigned char smr[];
  float* grouped = reinterpret_cast<float*>(smr);
  int* fill = reinterpret_cast<int*>(smr + (size_t)4 * T);   // exclusive prefix, then (after the scatter) bin ends
  unsigned* mixed = reinterpret_cast<unsigned*>(fill + K);  // bit b: bin b holds more than one value
  __shared__ float red_f[kRankWarps];
  __shared__ int red_i[kRankWarps];
  __shared__ long long red_l[kRankWarps];
  const int tid = threadIdx.x;
  const int64_t c = blockIdx.x;
  const float* src = xt + c * T;
  uint16_t* dst = rk + c * T;
  auto add_i = [](int a, int b) { return a + b; };
  // ---- sweep 1: valid count, finite min / max
  float mn = INFINITY, mx = -INFINITY;
  int n = 0;
  for (int t = tid; t < T; t += kRankThreads) {
    const float v = src[t];
    n += (v == v) ? 1 : 0;
    if (fabsf(v) < INFINITY) { mn = fminf(mn, v); mx = fmaxf(mx, v); }
  }
  n = block_reduce(n, add_i, red_i);
  mn = block_reduce(mn, [](float a, float b) { return fminf(a, b); }, red_f);
  mx = block_reduce(mx, [](float a, float b) { return fmaxf(a, b); }, red_f);
  float s = 0.f, o = 0.f;
  if (mx > mn) {
    const double sd = (double)(K - 3) / ((double)mx - (double)mn);
    s = (float)fmin(sd, (double)FLT_MAX);
    o = (float)(-(double)mn * (double)s);
  }
  for (int b = tid; b < K; b += kRankThreads) fill[b] = 0;
  for (int w = tid; w < K / 32; w += kRankThreads) mixed[w] = 0u;
  __syncthreads();
  // ---- sweep 2: histogram
  for (int t = tid; t < T; t += kRankThreads) {
    const float v = src[t];
    if (v == v) atomicAdd(&fill[bin_of<K>(v, s, o)], 1);
  }
  __syncthreads();
  block_exclusive_scan<K>(fill, red_i);
  __syncthreads();
  // ---- sweep 3: group the values by bin; fill[b] ends as the end of bin b, so bin b is [fill[b-1], fill[b])
  for (int t = tid; t < T; t += kRankThreads) {
    const float v = src[t];
    if (v == v) grouped[atomicAdd(&fill[bin_of<K>(v, s, o)], 1)] = v;
  }
  __syncthreads();
  auto bin_lo = [&](int b) { return b ? fill[b - 1] : 0; };
  for (int i = tid; i < n; i += kRankThreads) {
    const float v = grouped[i];
    const int b = bin_of<K>(v, s, o);
    if (v != grouped[bin_lo(b)]) atomicOr(&mixed[b >> 5], 1u << (b & 31));   // -0.0 == +0.0: one value
  }
  __syncthreads();
  long long cost = 0;
  for (int b = tid; b < K; b += kRankThreads) {
    if ((mixed[b >> 5] >> (b & 31)) & 1u) {
      const long long m = fill[b] - bin_lo(b);
      cost += m * m;
    }
  }
  cost = block_reduce(cost, [](long long a, long long b) { return a + b; }, red_l);
  int umin = INT_MAX, umax = -1;
  if (cost <= (long long)kCountBudget * n) {
    // ---- sweep 4: rank = (lower bins) + (own bin: below, equal)
    for (int t = tid; t < T; t += kRankThreads) {
      const float v = src[t];
      unsigned u = kNanRank;
      if (v == v) {
        const int b = bin_of<K>(v, s, o);
        const int lo = bin_lo(b), hi = fill[b];
        int less = 0, eq = hi - lo;
        if ((mixed[b >> 5] >> (b & 31)) & 1u) {
          eq = 0;
          for (int i = lo; i < hi; ++i) {
            const float w = grouped[i];
            less += (w < v) ? 1 : 0;
            eq += (w == v) ? 1 : 0;
          }
        }
        const int code = 2 * (lo + less) + eq - 1;
        umin = min(umin, code);
        umax = max(umax, code);
        u = (unsigned)code;
      }
      dst[t] = (uint16_t)u;
    }
  } else {
    // ---- sort the valid values (NaN -> +inf, padding +inf: the first n sorted keys are the valid values), then
    // rank by binary search; equal counts stop at n so that NaN and padding never tie with a real +inf
    float* keys = grouped;
    for (int t = tid; t < NPAD; t += kRankThreads) {
      const float v = (t < T) ? src[t] : INFINITY;
      keys[t] = (v == v) ? v : INFINITY;
    }
    __syncthreads();
    block_bitonic_sort<NPAD, kRankThreads>(keys, tid);
    for (int t = tid; t < T; t += kRankThreads) {
      const float v = src[t];
      unsigned u = kNanRank;
      if (v == v) {
        const int lo = lower_bound(keys, NPAD, v);
        const int hi = min(upper_bound(keys, NPAD, v), n);
        const int code = 2 * lo + (hi - lo) - 1;
        umin = min(umin, code);
        umax = max(umax, code);
        u = (unsigned)code;
      }
      dst[t] = (uint16_t)u;
    }
  }
  umin = block_reduce(umin, [](int a, int b) { return min(a, b); }, red_i);
  umax = block_reduce(umax, [](int a, int b) { return max(a, b); }, red_i);
  if (tid == 0) stats[c] = make_int4(n, n ? umin : 0, n ? umax : 0, 0);
}

// (3) 32 cells x rows_per_block steps per CTA (32 x 8 threads, lane = cell): rescale, factor, correction
template <int INTERP, int KIND>
__global__ void __launch_bounds__(kTile * 8, 2)
qdm_apply_kernel(const float* __restrict__ sim, int64_t T, int64_t ldx, int64_t nc, int64_t ldo,
                 const float* __restrict__ af, int64_t ldaf, const float* __restrict__ nodes, int32_t nq,
                 const uint16_t* __restrict__ rk, const int4* __restrict__ stats, int32_t rows_per_block,
                 float* __restrict__ scen, double* __restrict__ sim_q) {
  extern __shared__ float tabs[];   // [3][nq][32]: valid nodes, their af, nearest boundaries; column = cell
  float* xs = tabs;
  float* ys = xs + nq * kTile;
  float* bd = ys + nq * kTile;
  __shared__ int tile[kTile][kTile + 1];   // rank codes [cell][step]
  __shared__ int s_m[kTile];
  __shared__ double s_n[kTile], s_mn[kTile], s_mx[kTile];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int64_t cb = (int64_t)blockIdx.x * kTile;
  const int64_t c = cb + tx;
  const bool live = c < nc;
  if (ty == 0) {
    int m = 0;
    if (live) {
      for (int j = 0; j < nq; ++j) {   // interp1d on the entries where af is not NaN
        const float a = af[(int64_t)j * ldaf + c];
        if (a == a) { xs[m * kTile + tx] = nodes[j]; ys[m * kTile + tx] = a; ++m; }
      }
      for (int i = 0; i + 1 < m; ++i) bd[i * kTile + tx] = qmap::nearest_bound(xs[i * kTile + tx], xs[(i + 1) * kTile + tx]);
      const int4 st = stats[c];
      const double nd = (double)st.x;
      s_n[tx] = nd;
      s_mn[tx] = __ddiv_rn((double)(st.y + 2) * 0.5, nd);
      s_mx[tx] = __ddiv_rn((double)(st.z + 2) * 0.5, nd);
    }
    s_m[tx] = m;
  }
  __syncthreads();
  const int m = s_m[tx];
  const double nd = live ? s_n[tx] : 1.0, mn = live ? s_mn[tx] : 0.0, mx = live ? s_mx[tx] : 1.0;
  auto factor = [&](double q) -> float {
    float f;
    if (qmap::interp1d_edges<INTERP>(q, m, [&] { return xs[tx]; }, [&] { return xs[(m - 1) * kTile + tx]; },
                                     [&](int i) { return ys[i * kTile + tx]; }, f))
      return f;
    if (INTERP == 1) {
      // i = #{xs < q} clipped to [1, m - 1] (searchsorted side="left"): a guess from the uniform nodes, then
      // exact steps (more than one only where af had NaN entries)
      int i = min(max((int)(q * nq + 0.5), 1), m - 1);
      while (i > 1 && (double)xs[(i - 1) * kTile + tx] >= q) --i;
      while (i < m - 1 && (double)xs[i * kTile + tx] < q) ++i;
      const float x0 = xs[(i - 1) * kTile + tx], x1 = xs[i * kTile + tx];
      const float y0 = ys[(i - 1) * kTile + tx], y1 = ys[i * kTile + tx];
      return qmap::linear_two_weight(q, x0, x1, y0, y1);
    }
    // nearest: i = #{bd < q} (ties to the lower node) in [0, m - 1]
    int i = min(max((int)(q * nq), 0), m - 1);
    while (i > 0 && (double)bd[(i - 1) * kTile + tx] >= q) --i;
    while (i < m - 1 && (double)bd[i * kTile + tx] < q) ++i;
    return ys[i * kTile + tx];
  };
  const int64_t t0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t t1 = min(T, t0 + rows_per_block);
  for (int64_t tb = t0; tb < t1; tb += kTile) {
    float xv[kTile / 8];
#pragma unroll
    for (int k = 0; k < kTile / 8; ++k) {
      const int64_t t = tb + ty + 8 * k;
      xv[k] = (live && t < t1) ? ld_stream(sim + t * ldx + c) : 0.f;
    }
    for (int k = ty; k < kTile; k += 8) {   // ranks of 32 cells, read along time
      const int64_t cc = cb + k, t = tb + tx;
      tile[k][tx] = (cc < nc && t < t1) ? (int)rk[cc * T + t] : (int)kNanRank;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kTile / 8; ++k) {
      const int64_t t = tb + ty + 8 * k;
      if (!live || t >= t1) continue;
      const int u = tile[tx][ty + 8 * k];
      double q = NAN;
      if (u != (int)kNanRank) {
        const double p = __ddiv_rn((double)(u + 2) * 0.5, nd);                        // r / n, r = (u + 2) / 2
        q = __ddiv_rn(__dmul_rn(mx, __dsub_rn(p, mn)), __dsub_rn(mx, mn));            // (mx * (p - mn)) / (mx - mn)
      }
      const float f = factor(q);
      scen[t * ldo + c] = (KIND == 0) ? __fadd_rn(xv[k], f) : __fmul_rn(xv[k], f);
      if (sim_q) sim_q[t * ldo + c] = q;
    }
    __syncthreads();
  }
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int64_t xc_qdm_adjust_workspace_bytes(int64_t T, int64_t C) {
  T = T < 1 ? 1 : T;
  C = C < 1 ? 1 : C;
  return chunk_bytes(T, (C + kTile - 1) / kTile * kTile) + 256;
}

extern "C" int32_t xc_qdm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx, const float* af,
                                     const float* nodes, int32_t nq, int32_t kind, int32_t interp, float* scen,
                                     double* sim_q, void* workspace, int64_t workspace_bytes, void* stream) {
  XC_REQUIRE(sim && af && nodes && scen && workspace, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C, "bad shape");
  if (int32_t e = check_qmap_args(nq, 2, 200, kind, interp)) return e;
  XC_REQUIRE(C <= 2147483647LL, "too many cells for one launch");
  if (T > kMaxSteps) {
    set_error("qdm_adjust: series longer than 32768 steps do not fit the shared-memory ranking");
    return XC_ERR_UNSUPPORTED;
  }
  const int64_t need = xc_qdm_adjust_workspace_bytes(T, kTile);
  XC_REQUIRE(workspace_bytes >= need, "workspace too small: %lld bytes, at least %lld needed",
             (long long)workspace_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  // the largest chunk of whole 32-cell tiles that fits the workspace (256 bytes are kept for the alignment)
  char* base = reinterpret_cast<char*>(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  const int64_t avail = workspace_bytes - (int64_t)(base - reinterpret_cast<char*>(workspace));
  // (for whole tiles chunk_bytes(T, nc) is exactly nc * (6 T + 16))
  const int64_t all = (C + kTile - 1) / kTile * kTile;
  const int64_t cc = std::min(all, avail / (6 * T + 16) / kTile * kTile);
  size_t smem_rank = 0;
  auto rank = dispatch_npad(T, [&](auto NP) {
    constexpr int NPAD = decltype(NP)::value, K = NPAD / 4;
    smem_rank = std::max((size_t)4 * NPAD, (size_t)4 * T + (size_t)4 * K + (size_t)K / 8);
    return qdm_rank_kernel<NPAD>;
  });
  const size_t smem_apply = (size_t)3 * nq * kTile * 4;
  auto apply = dispatch_interp_kind(interp, kind, [](auto I, auto KD) { return qdm_apply_kernel<I.value, KD.value>; });
  if (int32_t e = allow_smem(rank, smem_rank, "cudaFuncSetAttribute(qdm_rank_kernel)")) return e;
  if (int32_t e = allow_smem(apply, smem_apply, "cudaFuncSetAttribute(qdm_apply_kernel)")) return e;
  for (int64_t c0 = 0; c0 < C; c0 += cc) {
    const int64_t nc = std::min(cc, C - c0);
    float* xt = reinterpret_cast<float*>(base);
    uint16_t* rk = reinterpret_cast<uint16_t*>(base + align16(nc * T * 4));
    int4* stats = reinterpret_cast<int4*>(base + align16(nc * T * 4) + align16(nc * T * 2));
    const unsigned tiles = (unsigned)((nc + kTile - 1) / kTile);
    qdm_transpose_kernel<<<dim3(tiles, (unsigned)((T + kTile - 1) / kTile)), dim3(kTile, 8), 0, st>>>(
        sim + c0, T, ldx, nc, xt);
    int32_t e = launch_status("qdm_transpose_kernel");
    if (e) return e;
    rank<<<(unsigned)nc, kRankThreads, smem_rank, st>>>(xt, (int32_t)T, rk, stats);
    e = launch_status("qdm_rank_kernel");
    if (e) return e;
    // time split: whole 32-row tiles, at least 4 of them per CTA
    const RowSplit split = split_rows(T, tiles, kTile, 4 * kTile);
    apply<<<dim3(tiles, (unsigned)split.chunks), dim3(kTile, 8), smem_apply, st>>>(
        sim + c0, T, ldx, nc, C, af + c0, C, nodes, nq, rk, stats, split.rows, scen + c0, sim_q ? sim_q + c0 : nullptr);
    e = launch_status("qdm_apply_kernel");
    if (e) return e;
  }
  return XC_OK;
}
