// Device rules shared by the quantile-mapping kernels: EQM train and adjust (eqm.cu), QDM apply (qdm.cu), DQM adjust
// and detrend (dqm.cu).
//
// dqm.cu is compiled with -fmad=false and the others with fused multiply-adds allowed.  The interpolation, position
// table and row-loop code that dqm.cu includes is explicit __f*_rn / __d*_rn rounding intrinsics, comparisons and
// integer arithmetic only, none of which -fmad touches, so it generates the same code in either file.  The train
// selection (numpy's _lerp included) is used by eqm.cu alone.
#pragma once
#include "common.cuh"

namespace xc {
namespace qmap {

// ---- train selection ----------------------------------------------------------------------------------------------
// node j of nq, cast to the data dtype before use (xsdba: equally_spaced_nodes(n).astype(ref.dtype))
__device__ __forceinline__ double node(int j, int nq) { return (double)(float)(((double)j + 0.5) / (double)nq); }

// rank of order statistic k of the 2 nq wanted among n valid values: quantile k / 2's floor(q (n - 1)) for an even k,
// the next rank (clipped to n - 1) for an odd one
__device__ __forceinline__ int target_rank(int k, int nq, int n) {
  const int ilo = (int)floor(node(k >> 1, nq) * (double)(n - 1));
  return (k & 1) ? min(ilo + 1, n - 1) : ilo;
}

// bin b with prefix(b) <= r < prefix(b + 1) among nbins bins, by bisection over the exclusive prefix sums
template <typename Prefix>
__device__ __forceinline__ int bin_of_rank(int r, int nbins, Prefix&& prefix) {
  int lo = 0, hi = nbins;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (prefix(mid) <= r) lo = mid; else hi = mid;
  }
  return lo;
}

// The values of ranks want0 and (TWO) want1 among the m candidates cl[] of one bin, ties ordered by position: the
// warp ranks them by counting and every lane gets the result (NaN for a rank not present).
template <bool TWO>
__device__ __forceinline__ float2 select_in_bin(const float* cl, int m, int want0, int want1, int lane) {
  float f0 = NAN, f1 = NAN;
  for (int i = lane; i < m; i += 32) {
    const float vi = cl[i];
    int less = 0;
    for (int k = 0; k < m; ++k) {
      const float vk = cl[k];
      less += (vk < vi || (vk == vi && k < i)) ? 1 : 0;
    }
    if (less == want0) f0 = vi;
    if (TWO && less == want1) f1 = vi;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float o0 = __shfl_xor_sync(0xffffffffu, f0, o);
    const float o1 = TWO ? __shfl_xor_sync(0xffffffffu, f1, o) : 0.f;
    f0 = (f0 == f0) ? f0 : o0;
    if (TWO) f1 = (f1 == f1) ? f1 : o1;
  }
  return make_float2(f0, f1);
}

// quantile j of n valid values from its two neighbouring order statistics v0, v1 (numpy's _lerp)
__device__ __forceinline__ float lerp_quantile(int j, int nq, int n, float v0, float v1) {
  const double pos = node(j, nq) * (double)(n - 1);
  const double g = pos - floor(pos);
  const double a0 = (double)v0, a1 = (double)v1;
  const double d = a1 - a0;
  return (float)((g >= 0.5) ? (a1 - d * (1.0 - g)) : (a0 + d * g));
}

// pass 0 (ref) keeps its quantile in refq; pass 1 (hist) writes hist_q and af = ref_q - hist_q ("+") or ref_q / hist_q
__device__ __forceinline__ void store_quantile(int pass, int32_t kind, float qv, float& refq, float* hist_q, float* af,
                                               int64_t at) {
  if (pass == 0) {
    refq = qv;
  } else {
    hist_q[at] = qv;
    af[at] = (kind == 0) ? (refq - qv) : (refq / qv);
  }
}

// ---- position table -----------------------------------------------------------------------------------------------
// #{keys < x} over the n sorted keys of a lane's shared-memory column (keys[j * NT]) without a bisection: NLUT bins of
// equal width over [first, first + range] (scale 0 when the range is not finite and positive: every value in bin 0),
// lut[b] = #{keys in a bin below b}.  The bins are a monotone function of the value, so a key in a lower bin is below
// x and lut[bin(x)] is a lower bound of the count; a forward scan while key < x finishes it.  K is the type the keys
// are compared in (float for EQM, double for DQM); UNROLL2 takes the first two scan steps unconditionally.
template <typename K, int NT, int NLUT, bool UNROLL2>
struct PosTable {
  const float* keys;    // this lane's column
  unsigned char* lut;   // this lane's column
  K first, scale;

  __device__ __forceinline__ PosTable(const float* keys_, unsigned char* lut_, K first_, K range, bool ok)
      : keys(keys_), lut(lut_), first(first_),
        scale((ok && range > K(0) && range < K(INFINITY)) ? K(NLUT) / range : K(0)) {}

  __device__ __forceinline__ int bin(K x) const {
    if constexpr (sizeof(K) == 4) {
      return max(0, min(NLUT - 1, (int)((x - first) * scale)));
    } else {
      const K b = (x - first) * scale;
      return b >= (K)(NLUT - 1) ? NLUT - 1 : (b > K(0) ? (int)b : 0);
    }
  }
  __device__ __forceinline__ K key(int j) const { return (K)keys[j * NT]; }

  // zero the table; then (fill) the histogram of the n keys' bins and its exclusive prefix
  __device__ __forceinline__ void build(int n, bool fill) const {
    for (int b = 0; b < NLUT; ++b) lut[b * NT] = 0;
    if (fill) {
      for (int j = 0; j < n; ++j) lut[bin(key(j)) * NT] += 1;
      int run = 0;
      for (int b = 0; b < NLUT; ++b) {
        const int c = lut[b * NT];
        lut[b * NT] = (unsigned char)run;
        run += c;
      }
    }
  }

  // #{keys < x} among n (searchsorted side="left")
  __device__ __forceinline__ int count_below(K x, int n) const {
    int i = lut[bin(x) * NT];
    if constexpr (UNROLL2) {
#pragma unroll
      for (int k = 0; k < 2; ++k) i += (i < n && key(min(i, n - 1)) < x) ? 1 : 0;
    }
    while (i < n && key(i) < x) ++i;
    return i;
  }
};

// ---- scipy interp1d on a compacted table (no NaN entries) ---------------------------------------------------------
// interp1d(kind="nearest")'s bound between neighbouring nodes: x_bds = x / 2; x_bds[1:] + x_bds[:-1], in float32
__device__ __forceinline__ float nearest_bound(float x0, float x1) {
  return __fadd_rn(__fmul_rn(x1, 0.5f), __fmul_rn(x0, 0.5f));
}

// interp1d(kind="linear")'s two-weight form ((x_new - x_lo) / dx) * y_hi + ((x_hi - x_new) / dx) * y_lo, dx = x_hi -
// x_lo in float32 (both nodes are float32), the rest in float64
__device__ __forceinline__ float linear_two_weight(double q, float x0, float x1, float y0, float y1) {
  const double dx = (double)__fsub_rn(x1, x0);
  const double w1 = __ddiv_rn(__dsub_rn(q, (double)x0), dx), w0 = __ddiv_rn(__dsub_rn((double)x1, q), dx);
  return __double2float_rn(__dadd_rn(__dmul_rn(w1, (double)y1), __dmul_rn(w0, (double)y0)));
}

// The cases decided before the search, on a table of m nodes: NaN for a NaN q or an empty table; with linear
// interpolation the fill values y(0) below x_first() and y(m - 1) above x_last(), and NaN at a one-node table's node
// (interp1d's slope 0 / 0).  Returns true with the factor in f when one of them applies.
template <int INTERP, typename XF, typename XL, typename Y>
__device__ __forceinline__ bool interp1d_edges(double q, int m, XF&& x_first, XL&& x_last, Y&& y, float& f) {
  if (!(q == q) || m == 0) { f = NAN; return true; }
  if (INTERP == 1) {
    if (q < (double)x_first()) { f = y(0); return true; }        // fill_value below
    if (q > (double)x_last()) { f = y(m - 1); return true; }     // ... and above
    if (m == 1) { f = NAN; return true; }
  }
  return false;
}

// ---- streaming rows -----------------------------------------------------------------------------------------------
// out[t * ldo] = f(in[t * ldx], t) for the rows [t0, t1) of one lane's column, U rows in flight
template <int U, typename TO, typename F>
__device__ __forceinline__ void stream_rows(const float* in, int64_t ldx, TO* out, int64_t ldo, int64_t t0, int64_t t1,
                                            F&& f) {
  int64_t t = t0;
  const float* ps = in + t0 * ldx;
  TO* po = out + t0 * ldo;
  for (; t + U <= t1; t += U) {
    float xv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) xv[u] = ld_stream(ps + (int64_t)u * ldx);
#pragma unroll
    for (int u = 0; u < U; ++u) po[(int64_t)u * ldo] = f(xv[u], t + u);
    ps += (int64_t)U * ldx;
    po += (int64_t)U * ldo;
  }
  for (; t < t1; ++t) {
    *po = f(ld_stream(ps), t);
    ps += ldx;
    po += ldo;
  }
}

}  // namespace qmap
}  // namespace xc
