// TEST INFRASTRUCTURE: a HOST build of the bootstrap mask reducer (xc::boot_reduce_year in
// xclim_b200/csrc/bootstrap_reduce_core.cuh), driven over every cell and in-base year as bootstrap_reduce_kernel
// does.  tests/test_bootstrap_reduce_host.py checks it against the oracle.  Nothing in xclim_b200/ loads it.
#include "../../xclim_b200/csrc/bootstrap_reduce_core.cuh"

// mask: [N (N - 1)][Wd][C] words; x: base rows (N * L, ldx); wet, out: (P, C), out float64 (COUNT / SPELL) or
// float32 (SUM)
extern "C" void boot_reduce_host(int red, const uint32_t* mask, int64_t C, int Wd, int N, int L,
                                 const int32_t* step_period, int window, int after, const float* x, int64_t ldx,
                                 const float* wet, void* out) {
  for (int y = 0; y < N; ++y)
    for (int64_t c = 0; c < C; ++c) {
      auto word = [&](int pair, int w) { return mask[((int64_t)pair * Wd + w) * C + c]; };
      auto xval = [&](int d) { return x[((int64_t)y * L + d) * ldx + c]; };
      auto wetp = [&](int p) { return wet[(int64_t)p * C + c]; };
      auto si = [&](int p, long long isum) { static_cast<double*>(out)[(int64_t)p * C + c] = xc::boot_int_mean(isum, N); };
      auto sf = [&](int p, double fsum, int nf) {
        static_cast<float*>(out)[(int64_t)p * C + c] = xc::boot_frac_mean(fsum, nf);
      };
      const int32_t* sp = step_period + (int64_t)y * L;
      if (red == XC_BOOT_COUNT)
        xc::boot_reduce_year<XC_BOOT_COUNT>(N, L, y, sp, window, after != 0, word, xval, wetp, si, sf);
      else if (red == XC_BOOT_SPELL)
        xc::boot_reduce_year<XC_BOOT_SPELL>(N, L, y, sp, window, after != 0, word, xval, wetp, si, sf);
      else
        xc::boot_reduce_year<XC_BOOT_SUM>(N, L, y, sp, window, after != 0, word, xval, wetp, si, sf);
    }
}
