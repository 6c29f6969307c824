// numpy's float32 pairwise summation (np.add.reduce over one contiguous run, which np.mean uses), for host and
// device.  Shared by the fire-weather day loop (fwi_core.cuh: means of <= 128 values) and the standardized-index
// fit (stdindex_core.cuh: means of a group's sample, of any length).  `at(k)` returns the k-th float32 value.
#pragma once

#if defined(__CUDACC__)
#define XC_NP_HD __host__ __device__ __forceinline__
#else
#define XC_NP_HD inline
#endif

namespace xc {
namespace np {

// One leaf of numpy's pairwise_sum, n <= 128: a plain loop below 8 values, else eight partial sums combined
// as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the n % 8 remaining values one by one.
template <class At>
XC_NP_HD float pairwise_block_f32(At at, int n) {
  float res;
  if (n < 8) {
    res = 0.0f;
    for (int k = 0; k < n; ++k) res += at(k);
  } else {
    float r[8];
    for (int j = 0; j < 8; ++j) r[j] = at(j);
    int k = 8;
    for (; k < n - (n % 8); k += 8)
      for (int j = 0; j < 8; ++j) r[j] += at(k + j);
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; k < n; ++k) res += at(k);
  }
  return res;
}

// The whole pairwise_sum: above 128 values numpy splits at n2 = n/2 - (n/2) % 8 and adds the two halves'
// sums.  The recursion is walked with an explicit stack (left subtree first, as numpy evaluates it); each
// split halves the length, so 24 frames cover every int length.
template <class At>
XC_NP_HD float pairwise_sum_f32(At at, int n) {
  if (n <= 128) return pairwise_block_f32(at, n);
  int right_off[24], right_n[24];
  float left[24];
  bool in_right[24];
  int sp = 0, off = 0, len = n;
  for (;;) {
    while (len > 128) {
      int n2 = len / 2;
      n2 -= n2 % 8;
      right_off[sp] = off + n2;
      right_n[sp] = len - n2;
      in_right[sp] = false;
      ++sp;
      len = n2;
    }
    const int base = off;
    float val = pairwise_block_f32([&](int k) { return at(base + k); }, len);
    for (;;) {
      if (sp == 0) return val;
      const int f = sp - 1;
      if (!in_right[f]) {
        left[f] = val;
        in_right[f] = true;
        off = right_off[f];
        len = right_n[f];
        break;
      }
      val = left[f] + val;
      --sp;
    }
  }
}

// x.mean() of n float32 values: the pairwise sum divided by n in float32 (NaN for n == 0).
template <class At>
XC_NP_HD float mean_f32(At at, int n) {
  return pairwise_sum_f32(at, n) / (float)n;
}

}  // namespace np
}  // namespace xc
