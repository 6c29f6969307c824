// Host build of the ensemble robustness device code (xclim_b200/csrc/ensemble_core.cuh) for the CPU test-suite:
// the Student-t distribution function and the two t-test p-values, compiled with g++ -ffp-contract=off.
#include <stdint.h>

#include "../../xclim_b200/csrc/ensemble_core.cuh"

using namespace xc::ens;

extern "C" {

void ens_host_stdtr(const double* df, const double* t, int64_t n, double* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = stdtr(df[i], t[i]);
}
double ens_host_ttest_1samp_p(int32_t n, double m, double ss, double popmean) {
  return ttest_1samp_p(n, m, ss, popmean);
}
double ens_host_welch_ttest_p(int32_t n1, double m1, double ss1, int32_t n2, double m2, double ss2) {
  return welch_ttest_p(n1, m1, ss1, n2, m2, ss2);
}

}  // extern "C"
