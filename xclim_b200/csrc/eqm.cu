// Empirical quantile mapping (sdba / xsdba `EmpiricalQuantileMapping`, group="time").
//
// The arithmetic lives in the third-party package xsdba (re-exported by sdba.py:11; floor pin
// xsdba>=0.4.0, pyproject.toml:111) whose sources are NOT under /root/reference: this file restates
// the published algorithm (PARITY UNPINNED, see DESIGN.md):
//   train : quantile nodes q_j = (j + 1/2)/nq; hist_q[j], ref_q[j] = NaN-aware linear (type 7)
//           quantiles of the whole series; af = ref_q - hist_q ("+") or ref_q / hist_q ("*").
//   adjust: scen = sim (+|*) interp(sim; hist_q -> af), nearest or linear, constant extrapolation.
// Reference call sites: tests/test_xsdba.py:21-34, 143-150.
//
// Design.  train needs ~2*nq order statistics spread over the WHOLE distribution of a
// 10950-sample series, i.e. a real per-cell sort: one CTA owns one cell, gathers its series into
// shared memory (64 KB for 16384 keys) and runs a bitonic sort there; neighbouring cells are
// handled by neighbouring CTAs at the same time so that the 32-byte sectors fetched by the strided
// gather are shared through L2.  adjust is a streaming pass: a lane owns one cell, keeps the 2*nq
// table entries of its cell in a conflict-free shared-memory column and does a binary search per
// element.
#include <stdlib.h>

#include "common.cuh"

namespace xc {
namespace {

#ifndef XC_EQM_THREADS
#define XC_EQM_THREADS 256
#endif
#ifndef XC_EQM_CAP
#define XC_EQM_CAP 128
#endif
constexpr int kSortThreads = XC_EQM_THREADS;
constexpr int kBins = 1024;      // histogram bins over [min, max] of the series
constexpr int kCap = XC_EQM_CAP; // candidates kept per needed bin
constexpr int kMaxTargets = 128; // order statistics per series (2 per quantile)

// Block-wide bitonic sort of keys[0..NPAD) ascending (fallback path).
template <int NPAD>
__device__ void block_bitonic_sort(float* keys, int tid) {
  for (int k = 2; k <= NPAD; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < NPAD / 2; i += kSortThreads) {
        const int a = ((i & ~(j - 1)) << 1) | (i & (j - 1));  // pair (a, a | j)
        const int b = a | j;
        const bool up = ((a & k) == 0);
        const float x0 = keys[a], x1 = keys[b];
        const bool swap = up ? (x0 > x1) : (x0 < x1);
        if (swap) { keys[a] = x1; keys[b] = x0; }
      }
      __syncthreads();
    }
  }
}

// One CTA = one cell.  The nq quantiles need only ~2*nq order statistics, so instead of sorting the
// series the CTA (1) histograms it over kBins equal-width bins between its min and max (binning by a
// monotone float expression keeps bins ordered), (2) locates the bin and the in-bin rank of every
// wanted order statistic from the prefix sums, (3) gathers only the elements of those bins and (4)
// ranks them by counting.  Degenerate distributions (a wanted bin with more than kCap elements that
// are not all equal, e.g. heavy ties next to other values) fall back to the full bitonic sort.
template <int NPAD>
__global__ void __launch_bounds__(kSortThreads)
eqm_train_kernel(const float* __restrict__ ref, const float* __restrict__ hist, int32_t T, int64_t C, int64_t ldx,
                 int32_t nq, int32_t kind, float* __restrict__ af, float* __restrict__ hist_q,
                 const int32_t* __restrict__ redo = nullptr) {
  extern __shared__ float keys[];             // NPAD keys | nq ref quantiles | candidate lists
  float* refq = keys + NPAD;
  float* cand = refq + ((nq + 3) & ~3);       // [2 * nq][kCap]
  __shared__ int hist_s[kBins + 1];           // counts, then exclusive prefix sums
  __shared__ int slot_of_bin[kBins];          // -1 or candidate-list slot
  __shared__ int cand_n[kMaxTargets];         // elements stored per slot
  __shared__ int tgt_rank[kMaxTargets], tgt_bin[kMaxTargets];
  __shared__ float tgt_val[kMaxTargets];
  __shared__ float red_min[kSortThreads / 32], red_max[kSortThreads / 32];
  __shared__ int red_cnt[kSortThreads / 32];
  __shared__ int s_flag, s_nslots;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int ntg = 2 * nq;
  // redo == nullptr: CTA = cell blockIdx.x.  Otherwise the CTAs walk the work list redo[1 .. redo[0]] (cells
  // eqm_train8_kernel could not finish); the trip count is uniform over the CTA.
  const int n_items = redo ? redo[0] : (int)gridDim.x;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x)
  for (int pass = 0; pass < 2; ++pass) {
    const int64_t c = redo ? (int64_t)redo[1 + item] : (int64_t)item;
    const float* src = (pass == 0 ? ref : hist) + c;
    // ---- load, count valid, min / max
    float mn = INFINITY, mx = -INFINITY;
    int nvalid = 0;
    for (int t = tid; t < T; t += kSortThreads) {
      const float v = ld_stream(src + (int64_t)t * ldx);
      keys[t] = v;
      if (v == v) { mn = fminf(mn, v); mx = fmaxf(mx, v); ++nvalid; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      nvalid += __shfl_xor_sync(0xffffffffu, nvalid, o);
    }
    if (lane == 0) { red_min[wid] = mn; red_max[wid] = mx; red_cnt[wid] = nvalid; }
    for (int b = tid; b <= kBins; b += kSortThreads) hist_s[b] = 0;
    for (int b = tid; b < kBins; b += kSortThreads) slot_of_bin[b] = -1;
    if (tid == 0) { s_flag = 0; s_nslots = 0; }
    __syncthreads();
    mn = red_min[0]; mx = red_max[0]; int n = 0;
    for (int w = 0; w < kSortThreads / 32; ++w) { mn = fminf(mn, red_min[w]); mx = fmaxf(mx, red_max[w]); n += red_cnt[w]; }
    const bool degenerate = !(mx > mn) || !(mx - mn < INFINITY);  // constant series, or infinite range
    const float scale = degenerate ? 0.f : (float)kBins / (mx - mn);
    auto bin_of = [&](float v) -> int { return min(kBins - 1, (int)((v - mn) * scale)); };
    bool use_sort = false;
    if (n > 0 && !degenerate) {
      // ---- histogram + prefix sums
      for (int t = tid; t < T; t += kSortThreads) {
        const float v = keys[t];
        if (v == v) atomicAdd(&hist_s[bin_of(v)], 1);
      }
      __syncthreads();
      if (wid == 0) {  // exclusive scan of kBins counters by one warp (kBins / 32 per lane)
        constexpr int per = kBins / 32;
        int loc[per], sum = 0;
#pragma unroll
        for (int i = 0; i < per; ++i) { loc[i] = hist_s[lane * per + i]; sum += loc[i]; }
        int incl = sum;
        for (int o = 1; o < 32; o <<= 1) {
          const int up = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += up;
        }
        int run = incl - sum;
#pragma unroll
        for (int i = 0; i < per; ++i) { hist_s[lane * per + i] = run; run += loc[i]; }
        if (lane == 31) hist_s[kBins] = run;
      }
      __syncthreads();
      // ---- wanted order statistics: ranks ilo, ihi of every quantile
      for (int g = tid; g < ntg; g += kSortThreads) {
        const int j = g >> 1;
        // nodes are cast to the data dtype before use (xsdba: equally_spaced_nodes(n).astype(ref.dtype))
        const double q = (double)(float)(((double)j + 0.5) / (double)nq);
        const int ilo = (int)floor(q * (double)(n - 1));
        const int r = (g & 1) ? min(ilo + 1, n - 1) : ilo;
        int lo = 0, hi = kBins;  // bin b with prefix[b] <= r < prefix[b+1]
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (hist_s[mid] <= r) lo = mid; else hi = mid;
        }
        tgt_bin[g] = lo;
        tgt_rank[g] = r - hist_s[lo];
        if (atomicCAS(&slot_of_bin[lo], -1, -2) == -1) {  // first to claim the bin allocates its slot
          const int sl = atomicAdd(&s_nslots, 1);
          cand_n[sl] = 0;
          slot_of_bin[lo] = sl;
        }
      }
      __syncthreads();
      // ---- gather the elements of the wanted bins
      for (int t = tid; t < T; t += kSortThreads) {
        const float v = keys[t];
        if (v == v) {
          const int sl = slot_of_bin[bin_of(v)];
          if (sl >= 0) {
            const int p = atomicAdd(&cand_n[sl], 1);
            if (p < kCap) cand[sl * kCap + p] = v;
          }
        }
      }
      __syncthreads();
      // ---- heavy bins (more than kCap elements): fine when all their elements are equal (ties, e.g. dry
      // days), which one extra block-wide min/max over that bin establishes; otherwise use the sort
      for (int sl = 0; sl < s_nslots; ++sl) {
        if (cand_n[sl] <= kCap) continue;  // uniform: shared memory value
        float lo_v = INFINITY, hi_v = -INFINITY;
        for (int t = tid; t < T; t += kSortThreads) {
          const float v = keys[t];
          if (v == v && slot_of_bin[bin_of(v)] == sl) { lo_v = fminf(lo_v, v); hi_v = fmaxf(hi_v, v); }
        }
        for (int o = 16; o > 0; o >>= 1) {
          lo_v = fminf(lo_v, __shfl_xor_sync(0xffffffffu, lo_v, o));
          hi_v = fmaxf(hi_v, __shfl_xor_sync(0xffffffffu, hi_v, o));
        }
        __syncthreads();  // red_* are free again
        if (lane == 0) { red_min[wid] = lo_v; red_max[wid] = hi_v; }
        __syncthreads();
        if (tid == 0) {
          float a = red_min[0], b = red_max[0];
          for (int w = 1; w < kSortThreads / 32; ++w) { a = fminf(a, red_min[w]); b = fmaxf(b, red_max[w]); }
          if (a == b) { cand[sl * kCap] = a; cand_n[sl] = -1; }  // constant bin
          else s_flag = 1;
        }
        __syncthreads();
      }
      // ---- rank inside the bin by counting (one warp per target)
      for (int g = wid; g < ntg; g += kSortThreads / 32) {
        const int sl = slot_of_bin[tgt_bin[g]];
        const int m = cand_n[sl];
        const float* cl = cand + sl * kCap;
        if (m < 0) {  // constant bin
          if (lane == 0) tgt_val[g] = cl[0];
          continue;
        }
        if (m > kCap) continue;  // resolved by the sort below
        const int want = tgt_rank[g];
        float found = NAN;
        for (int i = lane; i < m; i += 32) {
          const float vi = cl[i];
          int less = 0;
          for (int k = 0; k < m; ++k) {
            const float vk = cl[k];
            less += (vk < vi || (vk == vi && k < i)) ? 1 : 0;
          }
          if (less == want) found = vi;
        }
        for (int o = 16; o > 0; o >>= 1) {
          const float other = __shfl_xor_sync(0xffffffffu, found, o);
          found = (found == found) ? found : other;
        }
        if (lane == 0) tgt_val[g] = found;
      }
      __syncthreads();
      use_sort = (s_flag != 0);
    }
    if (use_sort) {
      // fallback: NaN -> +inf, pad with +inf, full sort; targets read from the sorted keys
      for (int t = tid; t < NPAD; t += kSortThreads) {
        float v = (t < T) ? keys[t] : INFINITY;
        if (v != v) v = INFINITY;
        keys[t] = v;
      }
      __syncthreads();
      block_bitonic_sort<NPAD>(keys, tid);
      for (int g = tid; g < ntg; g += kSortThreads) tgt_val[g] = keys[tgt_rank[g] + hist_s[tgt_bin[g]]];
      __syncthreads();
    }
    // ---- quantiles (numpy's _lerp on the two neighbours)
    for (int j = tid; j < nq; j += kSortThreads) {
      float qv = NAN;
      if (n > 0) {
        if (degenerate) {
          qv = mn;  // every valid value equals mn (or the range is not finite: not supported, gives mn)
        } else {
          const double q = (double)(float)(((double)j + 0.5) / (double)nq);
          const double pos = q * (double)(n - 1);
          const double lo = floor(pos);
          const double g = pos - lo;
          const double a0 = (double)tgt_val[2 * j], a1 = (double)tgt_val[2 * j + 1];
          const double d = a1 - a0;
          qv = (float)((g >= 0.5) ? (a1 - d * (1.0 - g)) : (a0 + d * g));
        }
      }
      if (pass == 0) {
        refq[j] = qv;
      } else {
        hist_q[(int64_t)j * C + c] = qv;
        af[(int64_t)j * C + c] = (kind == 0) ? (refq[j] - qv) : (refq[j] / qv);
      }
    }
    __syncthreads();
  }
}


// ------------------------------------------------------------------------------------------------
// train, a GROUP of adjacent cells per CTA: the same multi-select (min/max -> 1024-bin histogram -> gather the
// wanted bins -> rank by counting), but a CTA owns kG adjacent cells, i.e. kG * 4 contiguous bytes of every
// time row, and every fetched sector is used whole (the one-cell kernel fetched each sector for eight CTAs:
// 4 useful bytes per 32-byte sector).
//
// What bounds it: the number of (CTA, time row) TOUCHES.  At a 4 MB row stride every row of a CTA's slice
// lies in another DRAM page, and both earlier variants ran at the same rate of touches whatever the bytes per
// touch (16 cells x 3 sweeps: 4.3 G touches; 4 cells staged in shared memory x 1 sweep: 5.7 G touches, and
// slower by that ratio).  So the group is as WIDE as shared memory allows -- 32 cells = 128 bytes per touch --
// which needs the per-cell state small:
//   * the packed histogram (two 16-bit counters per word, T <= 32768) and the candidate pool share one
//     1024-word block per cell (the prefix sums are dead once the candidate offsets are known);
//   * bin -> slot is one byte per bin;
// and the sweeps short (they were ~30 instructions per element and sweep):
//   * bin = mantissa of fma(x - min, scale, 1.5 * 2^23): FADD + FFMA + IADD + VIMNMX, no F2I, no clamp pair;
//     a NaN lands in the extra bin kBins by the same unsigned min, so the histogram and the gather need no
//     branch on validity (bins are internal: any monotone binning yields the same order statistics);
//   * min / max by FMNMX alone (fminf / fmaxf drop NaN), the valid count is the histogram total.
// Candidate storage is allocated exactly from the histogram counts (prefix over the wanted bins).
// A cell this layout cannot finish -- a wanted bin with more than kHeavy elements that are not all equal,
// a candidate total beyond the pool, or a range so small that the scale overflows -- is appended to a redo
// list that the one-cell kernel resolves with its full machinery (sort fallback included): the results are
// those of eqm_train_kernel bit for bit.
// Instantiations: <32, 1024> default; <32, 512>; <16, 512> when C is a multiple of 16 only or the targets of
// 32 cells do not fit (nq > 40).
// ------------------------------------------------------------------------------------------------
constexpr int kPool = 1024;                 // candidate floats per cell (the same words hold the histogram first)
constexpr int kHeavy = 192;                 // bins above this must be constant
constexpr int kHistWords = kBins / 2 + 1;   // 512 words of two counters + the word of bin kBins (NaN sink)
constexpr int kClaimWord = kHistWords + 15; // 32 words of the block: one claim bit per bin (dead before the gather)
constexpr int kSobStride = kBins + 4;       // bin -> slot bytes per cell; entry kBins is never claimed
constexpr float kBinBias = 12582912.0f;     // 1.5 * 2^23: ulp 1 over [bias, bias + kBins]
constexpr int kBinBiasBits = 0x4B400000;
static_assert(kClaimWord + 32 <= kPool, "histogram + claim bits inside the cell's block");

__device__ __forceinline__ int float_key(float v) {   // order-preserving int key (for atomicMin / atomicMax)
  const int b = __float_as_int(v);
  return b >= 0 ? b : (b ^ 0x7fffffff);
}
__device__ __forceinline__ float key_float(int k) { return __int_as_float(k >= 0 ? k : (k ^ 0x7fffffff)); }

// bin of x: round((x - mn) * sc) for valid x (0 .. kBins - 1 since (mx - mn) * sc <= 1023 (1 + 2^-24)), kBins for NaN
__device__ __forceinline__ unsigned bin_index(float x, float mn, float sc) {
  const float t = fmaf(x - mn, sc, kBinBias);
  return min((unsigned)(__float_as_int(t) - kBinBiasBits), (unsigned)kBins);
}

// dynamic shared memory of eqm_train_group_kernel for ntg = 2 * nq targets per cell
__host__ __device__ inline size_t train_group_smem_bytes(int kG, int ntg) {
  return (size_t)kG * kPool * 4            // histogram / claim bits, then the candidate pool
         + (size_t)kG * kSobStride         // bin -> slot
         + (size_t)kG * ntg * (4 * 8);     // tgt_rank, tgt_bin, tgt_val, slot_bin, slot_off, slot_n, slot_min / max (2)
}

template <int kG, int kGT>
__global__ void __launch_bounds__(kGT, 1)
eqm_train_group_kernel(const float* __restrict__ ref, const float* __restrict__ hist, int32_t T, int64_t C,
                       int64_t ldx, int32_t nq, int32_t kind, float* __restrict__ af, float* __restrict__ hist_q,
                       int32_t* __restrict__ redo /* [0] = count, then cell indexes */) {
  extern __shared__ __align__(16) unsigned char smg[];
  const int ntg = 2 * nq;
  constexpr int kSub = kG / 4;       // threads (128-bit loads) per time row
  constexpr int kW = kGT / 32;
  static_assert(kG % 4 == 0 && kSub <= 16 && kGT % 32 == 0 && kW * 2 <= kPool, "layout");
  uint32_t* un = reinterpret_cast<uint32_t*>(smg);                            // [kG][kPool]
  unsigned char* sob = smg + (size_t)kG * kPool * 4;                          // [kG][kSobStride]
  int* tgt_rank = reinterpret_cast<int*>(sob + (size_t)kG * kSobStride);      // [kG][ntg]
  int* tgt_bin = tgt_rank + kG * ntg;
  float* tgt_val = reinterpret_cast<float*>(tgt_bin + kG * ntg);
  int* slot_bin = reinterpret_cast<int*>(tgt_val + kG * ntg);
  int* slot_off = slot_bin + kG * ntg;
  int* slot_n = slot_off + kG * ntg;
  int* slot_mm = slot_n + kG * ntg;                                           // [kG][ntg][2] min, max keys
  float* red_mn = reinterpret_cast<float*>(un);                               // [kW][kG], dead before the histogram
  float* red_mx = red_mn + kW * kG;
  __shared__ int nslots[kG], bad_cell[kG], cell_n[kG];
  __shared__ float cell_mn[kG], cell_scale[kG];
  __shared__ float refq[kG][64];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // thread = (time row mod kRows, 16-byte piece of the row): one 128-bit load covers 4 adjacent cells, kU loads in
  // flight per thread keep ~64 KB per SM on the wire
  const int half = tid % kSub, trow = tid / kSub;
  constexpr int kRows = kGT / kSub, kU = (kGT >= 1024) ? 4 : 8;
  const int64_t c0 = (int64_t)blockIdx.x * kG;
  constexpr unsigned kFree = 0xffu;
  auto pref_at = [&](int cc, int i) -> int {   // exclusive prefix sum of cell cc at bin i (i <= kBins)
    if (i >= kBins) return cell_n[cc];
    return (int)((un[cc * kPool + (i >> 1)] >> ((i & 1) * 16)) & 0xffffu);
  };
  // every sweep: f(v, u) on the float4 of row t for this thread's 4 cells
  auto sweep = [&](const float* src, auto&& f) {
    const int64_t step = (int64_t)kRows * ldx;
    const float* p = src + (int64_t)trow * ldx;
    int t = trow;
    for (; t + (kU - 1) * kRows < T; t += kU * kRows) {
      float4 v[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) v[u] = ld_stream4(p + u * step);
#pragma unroll
      for (int u = 0; u < kU; ++u) f(v[u]);
      p += kU * step;
    }
    for (; t < T; t += kRows) {
      f(ld_stream4(p));
      p += step;
    }
  };
  for (int pass = 0; pass < 2; ++pass) {
    const float* src = (pass == 0 ? ref : hist) + c0 + 4 * half;
    // ---- sweep 1: min, max of every cell (fminf / fmaxf drop NaN)
    {
      float mn4[4] = {INFINITY, INFINITY, INFINITY, INFINITY}, mx4[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
      sweep(src, [&](const float4& v) {
        mn4[0] = fminf(mn4[0], v.x); mx4[0] = fmaxf(mx4[0], v.x);
        mn4[1] = fminf(mn4[1], v.y); mx4[1] = fmaxf(mx4[1], v.y);
        mn4[2] = fminf(mn4[2], v.z); mx4[2] = fmaxf(mx4[2], v.z);
        mn4[3] = fminf(mn4[3], v.w); mx4[3] = fmaxf(mx4[3], v.w);
      });
      // lanes equal modulo kSub hold the same four cells
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int o = kSub; o < 32; o <<= 1) {
          mn4[i] = fminf(mn4[i], __shfl_xor_sync(0xffffffffu, mn4[i], o));
          mx4[i] = fmaxf(mx4[i], __shfl_xor_sync(0xffffffffu, mx4[i], o));
        }
        if (lane < kSub) { red_mn[wid * kG + 4 * lane + i] = mn4[i]; red_mx[wid * kG + 4 * lane + i] = mx4[i]; }
      }
    }
    __syncthreads();
    if (tid < kG) {
      float mn = INFINITY, mx = -INFINITY;
      for (int w = 0; w < kW; ++w) { mn = fminf(mn, red_mn[w * kG + tid]); mx = fmaxf(mx, red_mx[w * kG + tid]); }
      const bool degenerate = !(mx > mn) || !(mx - mn < INFINITY);
      float scale = degenerate ? 0.f : (float)(kBins - 1) / (mx - mn);
      const bool overflow = !(scale < INFINITY);       // a (sub)normal range: left to the one-cell kernel
      if (overflow) scale = 0.f;
      nslots[tid] = 0;
      bad_cell[tid] = overflow ? 1 : 0;
      cell_n[tid] = (mx >= mn) ? 1 : 0;                // any valid value; the histogram total replaces it below
      cell_mn[tid] = mn;
      cell_scale[tid] = scale;
    }
    __syncthreads();
    for (int cc = wid; cc < kG; cc += kW) {
      for (int w = lane; w < kClaimWord + 32; w += 32) un[cc * kPool + w] = 0u;
    }
    {
      uint32_t* sw = reinterpret_cast<uint32_t*>(sob);
      for (int i = tid; i < kG * kSobStride / 4; i += kGT) sw[i] = 0xffffffffu;
    }
    // the four cells this thread streams
    float cmn[4], csc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      cmn[i] = cell_mn[4 * half + i];
      csc[i] = cell_scale[4 * half + i];
    }
    __syncthreads();
    // ---- sweep 2: histogram (two 16-bit counters per word; a degenerate cell counts into bin 0, unused)
    {
      uint32_t* hb = un + (4 * half) * kPool;
      sweep(src, [&](const float4& v) {
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned b = bin_index(e[i], cmn[i], csc[i]);
          atomicAdd(hb + i * kPool + (b >> 1), 1u + (b & 1u) * 65535u);
        }
      });
    }
    __syncthreads();
    for (int cc = wid; cc < kG; cc += kW) {  // in-place exclusive scan of the kBins counters of cell cc by one warp
      constexpr int per = kBins / 32;
      uint32_t* hc = un + cc * kPool + lane * (per / 2);
      int loc[per], sum = 0;
#pragma unroll
      for (int i = 0; i < per; i += 2) {
        const uint32_t w2 = hc[i >> 1];
        loc[i] = (int)(w2 & 0xffffu);
        loc[i + 1] = (int)(w2 >> 16);
        sum += loc[i] + loc[i + 1];
      }
      int incl = sum;
      for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
      }
      int run = incl - sum;
#pragma unroll
      for (int i = 0; i < per; i += 2) {
        const uint32_t lo16 = (uint32_t)run;
        run += loc[i];
        const uint32_t hi16 = (uint32_t)run;
        run += loc[i + 1];
        hc[i >> 1] = lo16 | (hi16 << 16);
      }
      if (lane == 31 && cell_scale[cc] != 0.f) cell_n[cc] = run;   // the valid count
    }
    __syncthreads();
    // ---- wanted order statistics of every cell: bin + rank inside the bin; the first to want a bin gives it a slot
    for (int g = tid; g < kG * ntg; g += kGT) {
      const int cc = g / ntg, k = g - cc * ntg;
      const int nn = cell_n[cc];
      if (nn <= 0 || cell_scale[cc] == 0.f || c0 + cc >= C) continue;
      const int j = k >> 1;
      const double q = (double)(float)(((double)j + 0.5) / (double)nq);
      const int ilo = (int)floor(q * (double)(nn - 1));
      const int r = (k & 1) ? min(ilo + 1, nn - 1) : ilo;
      int lo = 0, hi = kBins;  // bin b with prefix[b] <= r < prefix[b+1]
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (pref_at(cc, mid) <= r) lo = mid; else hi = mid;
      }
      const int below = pref_at(cc, lo);
      tgt_bin[cc * ntg + k] = lo;
      tgt_rank[cc * ntg + k] = r - below;
      const uint32_t bit = 1u << (lo & 31);
      if (!(atomicOr(&un[cc * kPool + kClaimWord + (lo >> 5)], bit) & bit)) {
        const int sl = atomicAdd(&nslots[cc], 1);
        slot_bin[cc * ntg + sl] = lo;
        slot_off[cc * ntg + sl] = pref_at(cc, lo + 1) - below;     // the count; the offset after the next barrier
        slot_n[cc * ntg + sl] = 0;
        slot_mm[(cc * ntg + sl) * 2] = 0x7fffffff;
        slot_mm[(cc * ntg + sl) * 2 + 1] = (int)0x80000000;
        sob[cc * kSobStride + lo] = (unsigned char)sl;
      }
    }
    __syncthreads();
    // ---- candidate storage: exact offsets from the histogram counts (heavy bins are not gathered)
    if (tid < kG) {
      int off = 0;
      const int ns = nslots[tid];
      for (int sl = 0; sl < ns; ++sl) {
        const int cnt = slot_off[tid * ntg + sl];
        slot_off[tid * ntg + sl] = (cnt > kHeavy) ? -1 : off;
        if (cnt <= kHeavy) off += cnt;
      }
      if (off > kPool) {       // does not fit: nothing is gathered (min / max only) and the cell is redone
        bad_cell[tid] = 1;
        for (int sl = 0; sl < ns; ++sl) slot_off[tid * ntg + sl] = -1;
      }
    }
    __syncthreads();
    // ---- sweep 3: gather the elements of the wanted bins (min / max of the heavy ones)
    {
      const unsigned char* sb = sob + (4 * half) * kSobStride;
      sweep(src, [&](const float4& v) {
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const unsigned sl = sb[i * kSobStride + bin_index(e[i], cmn[i], csc[i])];
          if (sl != kFree) {
            const int cc = 4 * half + i;
            const int off = slot_off[cc * ntg + sl];
            if (off >= 0) {
              const int p = atomicAdd(&slot_n[cc * ntg + sl], 1);
              reinterpret_cast<float*>(un)[cc * kPool + off + p] = e[i];
            } else {
              const int kx = float_key(e[i]);
              atomicMin(&slot_mm[(cc * ntg + sl) * 2], kx);
              atomicMax(&slot_mm[(cc * ntg + sl) * 2 + 1], kx);
            }
          }
        }
      });
    }
    __syncthreads();
    // ---- heavy bins must be constant
    for (int g = tid; g < kG * ntg; g += kGT) {
      const int cc = g / ntg, sl = g - cc * ntg;
      if (sl < nslots[cc] && slot_off[cc * ntg + sl] < 0 &&
          slot_mm[(cc * ntg + sl) * 2] != slot_mm[(cc * ntg + sl) * 2 + 1])
        bad_cell[cc] = 1;
    }
    __syncthreads();
    // ---- rank inside the bin by counting: one warp per (cell, quantile); its two neighbours share the count
    // when they fall in the same bin
    for (int g = wid; g < kG * nq; g += kW) {
      const int cc = g / nq, j = g - cc * nq;
      if (cell_n[cc] <= 0 || cell_scale[cc] == 0.f || bad_cell[cc] || c0 + cc >= C) continue;
      const int k0 = cc * ntg + 2 * j;
      const int b0 = tgt_bin[k0], b1 = tgt_bin[k0 + 1];
      for (int h = 0; h < 2; ++h) {
        if (h == 1 && b1 == b0) break;
        const bool both = (h == 0 && b1 == b0);
        const int sl = sob[cc * kSobStride + (h ? b1 : b0)];
        const int off = slot_off[cc * ntg + sl];
        if (off < 0) {                                   // constant heavy bin
          if (lane == 0) {
            const float cv = key_float(slot_mm[(cc * ntg + sl) * 2]);
            tgt_val[k0 + h] = cv;
            if (both) tgt_val[k0 + 1] = cv;
          }
          continue;
        }
        const int m = slot_n[cc * ntg + sl];
        const float* cl = reinterpret_cast<const float*>(un) + cc * kPool + off;
        const int want0 = tgt_rank[k0 + h];
        const int want1 = both ? tgt_rank[k0 + 1] : -1;
        float f0 = NAN, f1 = NAN;
        for (int i = lane; i < m; i += 32) {
          const float vi = cl[i];
          int less = 0;
          for (int kk = 0; kk < m; ++kk) {
            const float vk = cl[kk];
            less += (vk < vi || (vk == vi && kk < i)) ? 1 : 0;
          }
          if (less == want0) f0 = vi;
          if (less == want1) f1 = vi;
        }
        for (int o = 16; o > 0; o >>= 1) {
          const float o0 = __shfl_xor_sync(0xffffffffu, f0, o);
          const float o1 = __shfl_xor_sync(0xffffffffu, f1, o);
          f0 = (f0 == f0) ? f0 : o0;
          f1 = (f1 == f1) ? f1 : o1;
        }
        if (lane == 0) {
          tgt_val[k0 + h] = f0;
          if (both) tgt_val[k0 + 1] = f1;
        }
      }
    }
    __syncthreads();
    // ---- quantiles (numpy's _lerp on the two neighbours)
    for (int g = tid; g < kG * nq; g += kGT) {
      const int cc = g / nq, j = g - cc * nq;
      if (c0 + cc >= C) continue;
      const int nn = cell_n[cc];
      float qv = NAN;
      if (nn > 0) {
        if (cell_scale[cc] == 0.f) {
          qv = cell_mn[cc];  // every valid value equals mn (or the range is not finite: not supported, gives mn)
        } else if (!bad_cell[cc]) {
          const double q = (double)(float)(((double)j + 0.5) / (double)nq);
          const double pos = q * (double)(nn - 1);
          const double lo = floor(pos);
          const double gq = pos - lo;
          const double a0 = (double)tgt_val[cc * ntg + 2 * j], a1 = (double)tgt_val[cc * ntg + 2 * j + 1];
          const double d = a1 - a0;
          qv = (float)((gq >= 0.5) ? (a1 - d * (1.0 - gq)) : (a0 + d * gq));
        }
      }
      if (pass == 0) {
        refq[cc][j] = qv;
      } else {
        hist_q[(int64_t)j * C + c0 + cc] = qv;
        af[(int64_t)j * C + c0 + cc] = (kind == 0) ? (refq[cc][j] - qv) : (refq[cc][j] / qv);
      }
    }
    __syncthreads();
    // a cell that could not be finished goes to the redo list (both passes are redone there)
    if (tid < kG && bad_cell[tid] && c0 + tid < C) {
      const int slot = atomicAdd(&redo[0], 1);
      redo[1 + slot] = (int)(c0 + tid);
    }
    __syncthreads();
  }
}


constexpr int kAdjThreads = 128;
constexpr int kLut = 32;   // coarse position table per cell

// adjust: a lane owns a cell and streams its series.  Per element the segment of the quantile table is found
// through a 32-entry position table of the cell instead of a 5-step bisection (~45 instructions per element,
// issue-bound): b = bin(x) on a uniform grid over [hq[0], hq[nq-1]],
// lut[b] = #{ j : bin(hq[j]) < b } is a LOWER bound of idx = #{ hq[j] < x } (bin() is monotone, so a node in a
// lower bin is below x), and the few nodes sharing x's bin are settled by a short forward scan -- two
// unconditional steps, then a loop that almost never runs.  Same idx, same arithmetic, bit-identical output.
template <int INTERP, int KIND>
__global__ void __launch_bounds__(kAdjThreads)
eqm_adjust_kernel(const float* __restrict__ sim, int64_t T, int64_t C, int64_t ldx, const float* __restrict__ af,
                  const float* __restrict__ hist_q, int32_t nq, int32_t rows_per_block, float* __restrict__ scen) {
  extern __shared__ float tab[];  // [3][nq][kAdjThreads]: hist_q, af, slope of the segment ending at j; column = lane
  float* hq = tab;
  float* fa = tab + (size_t)nq * kAdjThreads;
  float* sl = fa + (size_t)nq * kAdjThreads;
  unsigned char* lut = reinterpret_cast<unsigned char*>(sl + (size_t)nq * kAdjThreads);   // [kLut][kAdjThreads]
  const int lane = threadIdx.x;
  const int64_t c = (int64_t)blockIdx.x * kAdjThreads + lane;
  if (c >= C) return;
  bool bad = false;
  float hp = 0.f, ap = 0.f;
  for (int j = 0; j < nq; ++j) {
    const float h = hist_q[(int64_t)j * C + c], a = af[(int64_t)j * C + c];
    hq[j * kAdjThreads + lane] = h;
    fa[j * kAdjThreads + lane] = a;
    // the division of the linear interpolation is done once per segment instead of once per element
    // (same operands, same rounding: the results are bit-identical)
    sl[j * kAdjThreads + lane] = (j > 0) ? __fdiv_rn(__fsub_rn(a, ap), __fsub_rn(h, hp)) : 0.f;
    hp = h;
    ap = a;
    bad = bad || (h != h) || (a != a);
  }
  const int64_t t0 = (int64_t)blockIdx.y * rows_per_block;
  const int64_t t1 = min(T, t0 + rows_per_block);
  const float h_first = hq[lane], h_last = hq[(nq - 1) * kAdjThreads + lane];
  const float a_first = fa[lane], a_last = fa[(nq - 1) * kAdjThreads + lane];
  // position table (degenerate or non-finite ranges: scale 0 -> every x in bin 0 -> plain forward scan)
  const float range = h_last - h_first;
  const float scale = (!bad && range > 0.f && range < INFINITY) ? (float)kLut / range : 0.f;
  auto bin_of = [&](float x) -> int { return max(0, min(kLut - 1, (int)((x - h_first) * scale))); };
  for (int b = 0; b < kLut; ++b) lut[b * kAdjThreads + lane] = 0;
  if (!bad) {
    for (int j = 0; j < nq; ++j) {      // histogram of the nodes' bins, then exclusive prefix
      const int b = bin_of(hq[j * kAdjThreads + lane]);
      lut[b * kAdjThreads + lane] += 1;
    }
    int run = 0;
    for (int b = 0; b < kLut; ++b) {
      const int n = lut[b * kAdjThreads + lane];
      lut[b * kAdjThreads + lane] = (unsigned char)run;
      run += n;
    }
  }
  auto factor = [&](float x) -> float {
    if (bad || x != x) return NAN;
    if (x <= h_first) return a_first;
    if (x >= h_last) return a_last;
    // idx = #{hq < x} (searchsorted side="left"): lower bound from the table, forward scan inside the bin
    int idx = lut[bin_of(x) * kAdjThreads + lane];
#pragma unroll
    for (int k = 0; k < 2; ++k) idx += (idx < nq && hq[min(idx, nq - 1) * kAdjThreads + lane] < x) ? 1 : 0;
    while (idx < nq && hq[idx * kAdjThreads + lane] < x) ++idx;
    idx = max(1, min(idx, nq - 1));
    const float x0 = hq[(idx - 1) * kAdjThreads + lane];
    const float y0 = fa[(idx - 1) * kAdjThreads + lane];
    if (INTERP == 1) {
      const float slope = sl[idx * kAdjThreads + lane];
      return __fadd_rn(__fmul_rn(slope, __fsub_rn(x, x0)), y0);
    }
    // nearest: boundaries at the mid-points, ties go to the lower node
    const float x1 = hq[idx * kAdjThreads + lane], y1 = fa[idx * kAdjThreads + lane];
    const float mid = __fmul_rn(__fadd_rn(x0, x1), 0.5f);
    return (x <= mid) ? y0 : y1;
  };
  constexpr int U = 16;  // rows in flight per lane: shared memory caps the CTAs per SM at 6, so the bytes in flight come from here
  int64_t t = t0;
  const float* ps = sim + t0 * ldx + c;
  float* po = scen + t0 * C + c;
  for (; t + U <= t1; t += U) {
    float xv[U], fv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) xv[u] = ld_stream(ps + (int64_t)u * ldx);
#pragma unroll
    for (int u = 0; u < U; ++u) fv[u] = factor(xv[u]);
#pragma unroll
    for (int u = 0; u < U; ++u) po[(int64_t)u * C] = (KIND == 0) ? __fadd_rn(xv[u], fv[u]) : __fmul_rn(xv[u], fv[u]);
    ps += (int64_t)U * ldx;
    po += (int64_t)U * C;
  }
  for (; t < t1; ++t) {
    const float x = ld_stream(ps);
    const float f = factor(x);
    *po = (KIND == 0) ? __fadd_rn(x, f) : __fmul_rn(x, f);
    ps += ldx;
    po += C;
  }
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int64_t xc_eqm_train_workspace_bytes(int64_t T, int64_t C, int32_t nq) {
  (void)T; (void)nq;
  // redo list of the cell-group kernel: a counter + at most two entries per cell
  return 256 + (2 * C + 1) * 4;
}

// the one-cell-per-CTA kernel on `grid` CTAs: every cell (redo == nullptr, grid == C) or a work list
static int32_t launch_train_cells(const float* ref, const float* hist, int64_t T, int64_t C, int64_t ldx, int32_t nq,
                                  int32_t kind, float* af, float* hist_q, const int32_t* redo, unsigned grid,
                                  cudaStream_t st) {
  int npad = 1024;
  while (npad < T) npad <<= 1;
  const size_t smem = ((size_t)npad + ((nq + 3) & ~3) + (size_t)2 * nq * kCap) * 4;
#define XC_TRAIN(NP)                                                                                               \
  do {                                                                                                             \
    if (smem > 48 * 1024) {                                                                                        \
      cudaError_t e_ = cudaFuncSetAttribute(eqm_train_kernel<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                            (int)smem);                                                            \
      if (e_ != cudaSuccess) return cuda_fail(e_, "cudaFuncSetAttribute(eqm_train_kernel)");                       \
    }                                                                                                              \
    eqm_train_kernel<NP><<<grid, kSortThreads, smem, st>>>(ref, hist, (int32_t)T, C, ldx, nq, kind, af, hist_q,    \
                                                           redo);                                                  \
  } while (0)
  switch (npad) {
    case 1024: XC_TRAIN(1024); break;
    case 2048: XC_TRAIN(2048); break;
    case 4096: XC_TRAIN(4096); break;
    case 8192: XC_TRAIN(8192); break;
    case 16384: XC_TRAIN(16384); break;
    default: XC_TRAIN(32768); break;
  }
#undef XC_TRAIN
  return launch_status("eqm_train_kernel");
}

extern "C" int32_t xc_eqm_train_f32(const float* ref, const float* hist, int64_t T, int64_t C, int64_t ldx,
                                    int32_t nq, int32_t kind, float* af, float* hist_q, void* workspace,
                                    int64_t workspace_bytes, void* stream) {
  XC_REQUIRE(ref && hist && af && hist_q, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C, "bad shape");
  XC_REQUIRE(nq >= 1 && nq <= 64, "nquantiles must be in [1, 64]");
  XC_REQUIRE(kind == 0 || kind == 1, "kind must be 0 ('+') or 1 ('*')");
  XC_REQUIRE(C <= 2147483647LL, "too many cells for one launch");
  if (T > 32768) {
    set_error("eqm_train: series longer than 32768 steps do not fit the shared-memory sort");
    return XC_ERR_UNSUPPORTED;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t need = xc_eqm_train_workspace_bytes(T, C, nq);
  // widest group first: 32 cells = 128 bytes per (CTA, time row) touch; 16 when C is not a multiple of 32 or the
  // targets of 32 cells do not fit in shared memory.  (A variant that staged a 4-cell slice in shared memory and
  // read DRAM once was slower -- four times the row touches -- and is gone.)
  const char* kg_env = getenv("XCLIM_B200_EQM_KG");
  const char* gt_env = getenv("XCLIM_B200_EQM_GT");
  int g = 32;
  if (kg_env && atoi(kg_env) == 16) g = 16;
  if (g == 32 && (C % 32 != 0 || train_group_smem_bytes(32, 2 * nq) + 12 * 1024 > 227 * 1024)) g = 16;
  const bool fits = train_group_smem_bytes(g, 2 * nq) + 8 * 1024 <= 227 * 1024;
  const bool vec_ok = (C % g == 0) && (ldx % 4 == 0) && aligned16(ref) && aligned16(hist);
  if (workspace == nullptr || workspace_bytes < need || !vec_ok || !fits || getenv("XCLIM_B200_EQM_V1")) {
    // no scratch for a redo list, or a layout without whole 16-byte pieces per CTA: the one-cell-per-CTA
    // kernel (complete in itself)
    return launch_train_cells(ref, hist, T, C, ldx, nq, kind, af, hist_q, nullptr, (unsigned)C, st);
  }
  int32_t* redo = (int32_t*)workspace;
  XC_CHECK_CUDA(cudaMemsetAsync(redo, 0, 4, st));
  const size_t smemg = train_group_smem_bytes(g, 2 * nq);
  const int64_t groups = C / g;
#define XC_TRAIN_GROUP(G, GT)                                                                                      \
  do {                                                                                                             \
    XC_CHECK_CUDA(cudaFuncSetAttribute(eqm_train_group_kernel<G, GT>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                       (int)smemg));                                                               \
    eqm_train_group_kernel<G, GT><<<(unsigned)groups, GT, smemg, st>>>(ref, hist, (int32_t)T, C, ldx, nq, kind,   \
                                                                        af, hist_q, redo);                         \
  } while (0)
  if (g == 32 && gt_env && atoi(gt_env) == 512) XC_TRAIN_GROUP(32, 512);
  else if (g == 32) XC_TRAIN_GROUP(32, 1024);
  else XC_TRAIN_GROUP(16, 512);
#undef XC_TRAIN_GROUP
  int32_t e = launch_status("eqm_train_group_kernel");
  if (e) return e;
  // cells the eight-cell layout could not finish (heavy non-constant bins): a small fixed grid walks the list
  return launch_train_cells(ref, hist, T, C, ldx, nq, kind, af, hist_q, redo, 2u * (unsigned)sm_count(), st);
}

extern "C" int32_t xc_eqm_adjust_f32(const float* sim, int64_t T, int64_t C, int64_t ldx, const float* af,
                                     const float* hist_q, int32_t nq, int32_t kind, int32_t interp, float* scen,
                                     void* stream) {
  XC_REQUIRE(sim && af && hist_q && scen, "null pointer argument");
  XC_REQUIRE(T > 0 && C > 0 && ldx >= C, "bad shape");
  XC_REQUIRE(nq >= 2 && nq <= 200, "nquantiles must be in [2, 200]");   // node counts fit the 8-bit position table
  XC_REQUIRE(kind == 0 || kind == 1, "kind must be 0 ('+') or 1 ('*')");
  XC_REQUIRE(interp == 0 || interp == 1, "interp must be 0 (nearest) or 1 (linear)");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t cblocks = (C + kAdjThreads - 1) / kAdjThreads;
  int tchunks = (int)((sm_count() * 16 + cblocks - 1) / cblocks);
  tchunks = tchunks < 1 ? 1 : tchunks;
  int rows = (int)((T + tchunks - 1) / tchunks);
  if (rows < 64) rows = 64;
  tchunks = (int)((T + rows - 1) / rows);
  const size_t smem = (size_t)3 * nq * kAdjThreads * 4 + (size_t)kLut * kAdjThreads;
  dim3 grid((unsigned)cblocks, (unsigned)tchunks, 1);
#define XC_ADJ(I, K)                                                                                               \
  do {                                                                                                             \
    if (smem > 48 * 1024) {                                                                                        \
      cudaError_t e_ = cudaFuncSetAttribute(eqm_adjust_kernel<I, K>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                            (int)smem);                                                            \
      if (e_ != cudaSuccess) return cuda_fail(e_, "cudaFuncSetAttribute(eqm_adjust_kernel)");                      \
    }                                                                                                              \
    eqm_adjust_kernel<I, K><<<grid, kAdjThreads, smem, st>>>(sim, T, C, ldx, af, hist_q, nq, rows, scen);          \
  } while (0)
  if (interp == 0 && kind == 0) XC_ADJ(0, 0);
  else if (interp == 0) XC_ADJ(0, 1);
  else if (kind == 0) XC_ADJ(1, 0);
  else XC_ADJ(1, 1);
#undef XC_ADJ
  return launch_status("eqm_adjust_kernel");
}
