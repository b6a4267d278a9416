// numpy's np.add.reduce of a contiguous fp64 vector, restated in its summation order (dota_eval.cu, val_metrics.cu).
#pragma once
#include "common.cuh"

namespace y5obb {

// Pairwise summation with 8 partial sums up to 128 elements (the leaf) ...
__device__ inline double np_pairwise_leaf(const double* a, long long n) {
  if (n < 8) {
    double r = 0.0;
    for (long long i = 0; i < n; ++i) r = __dadd_rn(r, a[i]);
    return r;
  }
  double r[8];
  for (int j = 0; j < 8; ++j) r[j] = a[j];
  long long i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __dadd_rn(res, a[i]);
  return res;
}

// ... and above 128 sum(first n2) + sum(rest), n2 = n / 2 rounded down to a multiple of 8.  The recursion runs on an explicit
// frame array (at most 25 levels for n < 2^31), not the device call stack.
__device__ inline double np_pairwise_sum(const double* a, long long n) {
  struct Frame {
    long long off, n, n2;
    double left;
    int state;  // 0: not started, 1: left half pending, 2: right half pending
  };
  Frame st[32];
  int sp = 0;
  st[0] = {0, n, 0, 0.0, 0};
  double ret = 0.0;
  while (true) {
    Frame& f = st[sp];
    if (f.state == 0 && f.n <= 128) {
      ret = np_pairwise_leaf(a + f.off, f.n);
    } else if (f.state == 0) {
      f.n2 = f.n / 2 - (f.n / 2) % 8;
      f.state = 1;
      st[sp + 1] = {f.off, f.n2, 0, 0.0, 0};
      ++sp;
      continue;
    } else if (f.state == 1) {
      f.left = ret;
      f.state = 2;
      st[sp + 1] = {f.off + f.n2, f.n - f.n2, 0, 0.0, 0};
      ++sp;
      continue;
    } else {
      ret = __dadd_rn(f.left, ret);
    }
    if (sp == 0) return ret;
    --sp;
  }
}

}  // namespace y5obb
