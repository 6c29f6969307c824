// Host build of the standardized-index device code (xclim_b200/csrc/stdindex_core.cuh) for the CPU test-suite:
// the same special functions, per-cell fit and per-element transform, compiled with g++ -ffp-contract=off.
#include <stdint.h>

#include "../../xclim_b200/csrc/stdindex_core.cuh"

using namespace xc::si;

extern "C" {

void si_host_gammainc(const double* a, const double* x, int64_t n, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = gammainc(a[i], x[i]);
}
void si_host_digamma(const double* x, int64_t n, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = digamma(x[i]);
}
void si_host_ndtri(const double* p, int64_t n, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = ndtri(p[i]);
}
void si_host_ndtr(const double* z, int64_t n, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = ndtr(z[i]);
}
float si_host_np_mean(const float* v, int32_t n) {
  return xc::np::mean_f32([&](int k) { return v[k]; }, n);
}
double si_host_gamma_ml_shape(double s, double xa, double xb, int32_t* status) {
  int st = 0;
  const double a = gamma_ml_shape(s, xa, xb, &st);
  *status = st;
  return a;
}

// xc_si_fit_f32 on host arrays, cell by cell (workspace: max_n * C floats).
int32_t si_host_fit(const float* x, int64_t C, int64_t ldx, const int32_t* goff, const int32_t* steps, int32_t G,
                    int32_t dist, int32_t method, int32_t zi, double floc, double* params, int32_t* n_zeros,
                    int32_t* n_notnull, float* ws) {
  int st = 0;
  for (int64_t c = 0; c < C; ++c)
    st |= fit_cell(x, C, ldx, c, goff, steps, G, dist, method, zi, floc, params, zi ? n_zeros : nullptr,
                   zi ? n_notnull : nullptr, ws + c);
  return st;
}

// xc_si_apply_f32 on host arrays.
void si_host_apply(const float* x, int64_t T, int64_t C, int64_t ldx, const int16_t* gos, const double* params,
                   const int32_t* n_zeros, const int32_t* n_notnull, int32_t dist, int32_t zi, double interp,
                   double alpha, double beta, double* out) {
  for (int64_t t = 0; t < T; ++t)
    for (int64_t c = 0; c < C; ++c) {
      const int g = gos[t];
      double r = NAN;
      if (g >= 0) {
        const double* p = params + (int64_t)g * 3 * C + c;
        r = standardized(dist, x[t * ldx + c], p[0], p[C], p[2 * C], zi != 0, zi ? n_zeros[(int64_t)g * C + c] : 0,
                         zi ? n_notnull[(int64_t)g * C + c] : 0, interp, alpha, beta);
      }
      out[t * C + c] = r;
    }
}

}  // extern "C"
