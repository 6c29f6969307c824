// Spatial analogues on the device: the dissimilarity between each target sample and every candidate cell
// (xc_analog_f32, include/xclim_b200.h a1).
//
// Replaces analog.py `spatial_analogs` (:87-97), where every cell is one numpy / scipy call inside
// xr.apply_ufunc(vectorize=True).  The arithmetic lives in analog_core.cuh, which the CPU test-suite also
// compiles for the host; this file adds the thread mapping and the argument checks.
//
// One CTA per (32-cell tile, target).  Its 256 threads copy the tile's m * d candidate rows into shared memory as
// whole 128-byte row segments (row r of the tile at r * 33 floats: padded, so a lane reading its own indicator
// hits its own bank), and the target sample as float64.  Each warp then takes cells j = warp, warp + 8, ... of
// the tile, and its lanes split the O((n + m)^2) pair loops by their first point; float64 partials meet in
// an xor-shuffle butterfly that the host build repeats addition for addition.  kldiv and nearest_neighbor keep
// their neighbour lists in registers, kolmogorov_smirnov the pooled quadrant codes of the current pivot in the
// warp's shared scratch.  Built with -fmad=false, like the host build's -ffp-contract=off.
#include "common.cuh"
#include "analog_core.cuh"

namespace xc {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kTile = 32;
constexpr int kRow = kTile + 1;      // padded row of a tile in shared memory
constexpr int kStats = 5;            // per warp: mean_x, std_x, mean_y, std_y, and the per-indicator scale

int64_t n_consts(int method, int64_t d) {
  return method == an::kSeuclidean ? d : method == an::kMaha ? d * d : 0;
}

// shared memory: target (n d) | consts | per-warp stats (kWarps 5 d) as float64, per-warp codes (kWarps (n + m))
// as uint32, candidate tile (m d kRow) as float32
int64_t smem_bytes(int64_t n, int64_t m, int64_t d, int64_t nc) {
  return 8 * (n * d + nc + kWarps * kStats * d) + 4 * kWarps * (n + m) + 4 * m * d * kRow;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

// pivot(A, B) of kolmogorov_smirnov over the pool A then B
template <class Pool>
__device__ double ks_pivot(Pool P, int nA, int nB, int d, uint32_t* codes, int lane) {
  double best = 0.0;
  for (int b = 0; b < nA; ++b) {
    for (int a = lane; a < nA + nB; a += 32) codes[a] = an::ks_code(P, b, a, d);
    __syncwarp();
    best = fmax(best, an::ks_diff(codes, nA, nB, lane, 32));
    __syncwarp();
  }
  return warp_max(best);
}

template <int DB>
__device__ double analog_cell(const double* xs, const float* yc, int n, int m, int d, int method, double param,
                              const double* cst, double* st, uint32_t* codes, int lane, int32_t* status) {
  auto X = [&](int i, int k) { return xs[i * d + k]; };
  auto Y = [&](int s, int k) { return (double)yc[(s * d + k) * kRow]; };
  auto P = [&](int p, int k) { return p < n ? X(p, k) : Y(p - n, k); };
  bool nan = false;
  for (int i = lane; i < n * d; i += 32) nan |= isnan(xs[i]);
  for (int i = lane; i < m * d; i += 32) nan |= isnan(yc[i * kRow]);
  if (__any_sync(0xffffffffu, nan)) return NAN;

  double *mx = st, *sx = st + d, *my = st + 2 * d, *sy = st + 3 * d, *v = st + 4 * d;
  if (lane < d) {
    an::col_stats(X, n, lane, mx + lane, sx + lane);
    an::col_stats(Y, m, lane, my + lane, sy + lane);
    v[lane] = method == an::kNearest ? sqrt(sx[lane] * sy[lane]) : sx[lane] * sy[lane];
  }
  __syncwarp();

  double r = NAN;
  if (method == an::kSeuclidean) {
    bool bad = false;
    r = an::seuclidean(mx, my, cst, d, &bad);
    if (bad && lane == 0) atomicOr(status, XC_AN_STATUS_CHKFINITE);
  } else if (method == an::kMaha) {
    r = an::mahalanobis(mx, my, cst, d);
  } else if (method == an::kZech || method == an::kSzekely) {
    const bool zech = method == an::kZech;
    double s[3];
    an::pair_sums<DB>(P, n, m, d, zech || param != 0.0 ? v : nullptr, zech, param, lane, 32, s);
    for (int t = 0; t < 3; ++t) s[t] = warp_sum(s[t]);
    r = zech ? an::zech_finish(s, n, m) : an::szekely_finish(s, n, m);
  } else if (method == an::kNearest) {
    bool bad = false;
    for (int i = lane; i < (n + m) * d; i += 32) bad |= !isfinite(P(i / d, i % d) / v[i % d]);
    if (__any_sync(0xffffffffu, bad)) {
      if (lane == 0) atomicOr(status, XC_AN_STATUS_NOT_FINITE);
      return NAN;
    }
    r = (double)warp_sum(an::nn_count<DB>(P, n, m, d, v, lane, 32)) / (n + m);
  } else if (method == an::kKs) {
    auto Q = [&](int p, int k) { return p < m ? Y(p, k) : X(p - m, k); };
    const double pxy = ks_pivot(P, n, m, d, codes, lane);
    const double pyx = ks_pivot(Q, m, n, d, codes, lane);
    r = pxy >= pyx ? pxy : pyx;
  } else if (method == an::kKldiv) {
    if (n < 5 || m < 5) return NAN;
    bool bad = false;
    for (int i = lane; i < (n + m) * d; i += 32) bad |= isinf(P(i / d, i % d));
    if (__any_sync(0xffffffffu, bad)) {
      if (lane == 0) atomicOr(status, XC_AN_STATUS_NOT_FINITE);
      return NAN;
    }
    const int k = (int)param;
    const double part = k <= 1 ? an::kl_partial<DB, 2>(P, n, m, d, k, lane, 32)
                               : an::kl_partial<DB, XC_AN_KLDIV_MAX_K + 1>(P, n, m, d, k, lane, 32);
    r = an::kl_finish(warp_sum(part), n, m, d);
  }
  return r;
}

template <int DB>
__global__ void __launch_bounds__(kThreads)
analog_kernel(const float* __restrict__ target, int n, const float* __restrict__ cand, int m, int64_t C,
              int64_t ldc, int d, int method, double param, const double* __restrict__ consts, int nc,
              double* __restrict__ out, int32_t* __restrict__ status) {
  extern __shared__ double smem[];
  double* xs = smem;
  double* cst = xs + n * d;
  double* stats = cst + nc;
  uint32_t* codes = (uint32_t*)(stats + kWarps * kStats * d);
  float* ys = (float*)(codes + kWarps * (n + m));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.y;
  const int64_t c0 = (int64_t)blockIdx.x * kTile;
  const int width = (int)(C - c0 < kTile ? C - c0 : kTile);

  for (int i = threadIdx.x; i < n * d; i += kThreads) xs[i] = target[(int64_t)t * n * d + i];
  for (int i = threadIdx.x; i < nc; i += kThreads) cst[i] = consts[(int64_t)t * nc + i];
  for (int r = warp; r < m * d; r += kWarps)
    ys[r * kRow + lane] = lane < width ? __ldg(cand + r * ldc + c0 + lane) : 0.0f;
  __syncthreads();

  for (int j = warp; j < width; j += kWarps) {
    const double res = analog_cell<DB>(xs, ys + j, n, m, d, method, param, cst, stats + warp * kStats * d,
                                       codes + warp * (n + m), lane, status);
    if (lane == 0) out[(int64_t)t * C + c0 + j] = res;
    __syncwarp();
  }
}

template <int DB>
int32_t launch(const float* target, int64_t n, int64_t K, const float* cand, int64_t m, int64_t C, int64_t ldc,
               int64_t d, int32_t method, double param, const double* consts, int64_t nc, double* out,
               int32_t* status, int64_t smem, cudaStream_t stream) {
  XC_CHECK_CUDA(cudaFuncSetAttribute(analog_kernel<DB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)((C + kTile - 1) / kTile), (unsigned)K, 1);
  analog_kernel<DB><<<grid, kThreads, smem, stream>>>(target, (int)n, cand, (int)m, C, ldc, (int)d, method, param,
                                                       consts, (int)nc, out, status);
  return launch_status("analog_kernel");
}

}  // namespace
}  // namespace xc

using namespace xc;

extern "C" int32_t xc_analog_f32(const float* target, int64_t n, int64_t K, const float* cand, int64_t m, int64_t C,
                                 int64_t ldc, int64_t d, int32_t method, double param, const double* consts,
                                 double* out, int32_t* status, void* stream) {
  XC_REQUIRE(target && cand && out && status, "null pointer argument");
  XC_REQUIRE(method >= an::kSeuclidean && method <= an::kMaha, "unknown analogue method %d", method);
  XC_REQUIRE(n > 0 && m > 0 && K > 0 && K <= 65535 && C > 0 && ldc >= C, "bad shape");
  XC_REQUIRE(d > 0 && d <= XC_AN_MAX_D, "the number of indicators must be in [1, %d], got %lld", XC_AN_MAX_D,
             (long long)d);
  const int64_t nc = n_consts(method, d);
  XC_REQUIRE(nc == 0 || consts, "seuclidean and mahalanobis need their per-target constants");
  if (method == an::kKldiv) {
    XC_REQUIRE(d <= 10, "Too many dimensions: %lld.", (long long)d);
    XC_REQUIRE(param >= 1 && param <= XC_AN_KLDIV_MAX_K && param == (double)(int)param,
               "kldiv needs an integer k in [1, %d]", XC_AN_KLDIV_MAX_K);
  }
  const int64_t smem = smem_bytes(n, m, d, nc);
  XC_REQUIRE(n * d <= (1 << 20) && m * d <= (1 << 20) && smem <= 227 * 1024,
             "samples of %lld and %lld points of %lld indicators need %lld bytes of shared memory per block: too large",
             (long long)n, (long long)m, (long long)d, (long long)smem);
  if (d <= 4)
    return launch<4>(target, n, K, cand, m, C, ldc, d, method, param, consts, nc, out, status, smem,
                     (cudaStream_t)stream);
  return launch<XC_AN_MAX_D>(target, n, K, cand, m, C, ldc, d, method, param, consts, nc, out, status, smem,
                             (cudaStream_t)stream);
}
