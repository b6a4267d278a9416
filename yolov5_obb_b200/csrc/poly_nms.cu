// Tile-merge polygon NMS of the DOTA devkit on the device (SURVEY section 8f rank 4, row A14's CPU form):
//   DOTA_devkit/ResultMerge_multi_process.py:62-123  py_cpu_nms_poly_fast
//   DOTA_devkit/polyiou.cpp:9-128                    iou_poly (double, eps = 1e-8 sign tests)
// Written against the bit-equal CPU restatement (oracle/poly_ref.py, pinned to the reference's polyiou.cpp compiled in
// place); tests/test_poly_gpu.py checks the IoUs bit-equal and the keep lists equal to the reference's.
//
// Pipeline: CUB radix sort by descending score (stable, ties -> lower index, as numpy's argsort()[::-1] is NOT: the
// reference's tie order is the reverse index order; callers with tied scores get the documented lower-index-first rule) ->
// k_poly_mask: for every pair i < j of the sorted order the axis-aligned pre-filter and, where it fires, the polygon IoU
// in double precision with explicit round-to-nearest multiplies / adds (no FMA contraction: bit-equal to the reference's
// g++ -O2 build) -> bit r of word (i, j / 64) = "j is suppressed by i" = !(ovr <= thresh) -> k_poly_reduce: greedy scan.
#include <cub/cub.cuh>

#include "common.cuh"

namespace y5obb {
namespace {

constexpr double PEPS = 1e-8;

struct P2 {
  double x, y;
};

__device__ __forceinline__ int psig(double d) { return (d > PEPS) - (d < -PEPS); }
__device__ __forceinline__ double pmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double padd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double psub(double a, double b) { return __dsub_rn(a, b); }
// (a.x-o.x)*(b.y-o.y) - (b.x-o.x)*(a.y-o.y)
__device__ __forceinline__ double pcross(P2 o, P2 a, P2 b) {
  return psub(pmul(psub(a.x, o.x), psub(b.y, o.y)), pmul(psub(b.x, o.x), psub(a.y, o.y)));
}
__device__ double parea(const P2* ps, int n) {
  double res = 0.0;
  for (int i = 0; i < n; ++i) {
    const int j = (i + 1 == n) ? 0 : i + 1;
    res = padd(res, psub(pmul(ps[i].x, ps[j].y), pmul(ps[i].y, ps[j].x)));
  }
  return res / 2.0;
}
__device__ __forceinline__ bool psame(P2 p, P2 q) { return psig(psub(p.x, q.x)) == 0 && psig(psub(p.y, q.y)) == 0; }

// polyiou.cpp:57-70: the part of polygon p (n points, n <= 8) to the left of a->b, in place
__device__ void polygon_cut(P2* p, int& n, P2 a, P2 b) {
  P2 pp[12];
  int m = 0;
  for (int i = 0; i < n; ++i) {
    const P2 pi = p[i], pj = p[(i + 1 == n) ? 0 : i + 1];
    const int si = psig(pcross(a, b, pi)), sj = psig(pcross(a, b, pj));
    if (si > 0) pp[m++] = pi;
    if (si != sj) {
      const double s1 = pcross(a, b, pi), s2 = pcross(a, b, pj);
      P2 x = pi;  // lineCross leaves its output untouched for (anti)parallel lines: cannot happen when the signs differ
      if (!(psig(s1) == 0 && psig(s2) == 0) && psig(psub(s2, s1)) != 0) {
        const double d = psub(s2, s1);
        x.x = psub(pmul(pi.x, s2), pmul(pj.x, s1)) / d;
        x.y = psub(pmul(pi.y, s2), pmul(pj.y, s1)) / d;
      }
      pp[m++] = x;
    }
  }
  n = 0;
  for (int i = 0; i < m; ++i)
    if (i == 0 || !psame(pp[i], pp[i - 1])) p[n++] = pp[i];
  while (n > 1 && psame(p[n - 1], p[0])) --n;
}

// polyiou.cpp:73-88: signed intersection area of the triangles (o, a, b) and (o, c, d), o the origin
__device__ double tri_intersect(P2 a, P2 b, P2 c, P2 d) {
  const P2 o = {0.0, 0.0};
  const int s1 = psig(pcross(o, a, b)), s2 = psig(pcross(o, c, d));
  if (s1 == 0 || s2 == 0) return 0.0;
  if (s1 == -1) {
    const P2 t = a;
    a = b;
    b = t;
  }
  if (s2 == -1) {
    const P2 t = c;
    c = d;
    d = t;
  }
  P2 p[12];
  p[0] = o;
  p[1] = a;
  p[2] = b;
  int n = 3;
  polygon_cut(p, n, o, c);
  polygon_cut(p, n, c, d);
  polygon_cut(p, n, d, o);
  const double res = n > 0 ? fabs(parea(p, n)) : 0.0;
  return (s1 * s2 == -1) ? -res : res;
}

__device__ double iou_poly_dev(const double* p8, const double* q8) {
  P2 a[4], b[4];
  for (int i = 0; i < 4; ++i) {
    a[i].x = p8[2 * i];
    a[i].y = p8[2 * i + 1];
    b[i].x = q8[2 * i];
    b[i].y = q8[2 * i + 1];
  }
  if (parea(a, 4) < 0) {
    P2 t = a[0];
    a[0] = a[3];
    a[3] = t;
    t = a[1];
    a[1] = a[2];
    a[2] = t;
  }
  if (parea(b, 4) < 0) {
    P2 t = b[0];
    b[0] = b[3];
    b[3] = t;
    t = b[1];
    b[1] = b[2];
    b[2] = t;
  }
  double inter = 0.0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) inter = padd(inter, tri_intersect(a[i], a[(i + 1) & 3], b[j], b[(j + 1) & 3]));
  const double uni = psub(padd(fabs(parea(a, 4)), fabs(parea(b, 4))), inter);
  return inter / uni;
}

__global__ void k_poly_keys(const double* __restrict__ dets9, long long n, unsigned long long* __restrict__ keys,
                            unsigned int* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long u = (unsigned long long)__double_as_longlong(dets9[i * 9 + 8] + 0.0);
  u ^= (u >> 63) ? ~0ull : 0x8000000000000000ull;  // ascending on unsigned compare
  keys[i] = ~u;                                      // descending score
  vals[i] = (unsigned int)i;
}

__global__ void k_poly_pair_iou(const double* __restrict__ p8, const double* __restrict__ q8, double* __restrict__ out,
                                long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = iou_poly_dev(p8 + 8 * i, q8 + 8 * i);
}

// one thread per (row i, 64-column word): bit c = candidate (w * 64 + c) of the sorted order is suppressed by i
__global__ void k_poly_mask(const double* __restrict__ dets9, const unsigned int* __restrict__ order, long long n, double thresh,
                            unsigned long long* __restrict__ mask) {
  const long long words = (n + 63) / 64;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * words) return;
  const long long i = t / words, w = t - i * words;
  unsigned long long bits = 0ull;
  if ((w + 1) * 64 > i + 1) {
    const double* di = dets9 + (long long)order[i] * 9;
    double ix1 = di[0], ix2 = di[0], iy1 = di[1], iy2 = di[1];
    for (int k = 1; k < 4; ++k) {
      ix1 = fmin(ix1, di[2 * k]);
      ix2 = fmax(ix2, di[2 * k]);
      iy1 = fmin(iy1, di[2 * k + 1]);
      iy2 = fmax(iy2, di[2 * k + 1]);
    }
    const double ai = pmul(padd(psub(ix2, ix1), 1.0), padd(psub(iy2, iy1), 1.0));
    for (int c = 0; c < 64; ++c) {
      const long long j = w * 64 + c;
      if (j <= i || j >= n) continue;
      const double* dj = dets9 + (long long)order[j] * 9;
      double jx1 = dj[0], jx2 = dj[0], jy1 = dj[1], jy2 = dj[1];
      for (int k = 1; k < 4; ++k) {
        jx1 = fmin(jx1, dj[2 * k]);
        jx2 = fmax(jx2, dj[2 * k]);
        jy1 = fmin(jy1, dj[2 * k + 1]);
        jy2 = fmax(jy2, dj[2 * k + 1]);
      }
      const double aj = pmul(padd(psub(jx2, jx1), 1.0), padd(psub(jy2, jy1), 1.0));
      const double ww = fmax(0.0, psub(fmin(ix2, jx2), fmax(ix1, jx1)));
      const double hh = fmax(0.0, psub(fmin(iy2, jy2), fmax(iy1, jy1)));
      const double hb = pmul(ww, hh);
      double ovr = hb / psub(padd(ai, aj), hb);
      if (ovr > 0) ovr = iou_poly_dev(di, dj);
      if (!(ovr <= thresh)) bits |= 1ull << c;
    }
  }
  mask[i * words + w] = bits;
}

__global__ void k_poly_reduce(const unsigned long long* __restrict__ mask, const unsigned int* __restrict__ order, long long n,
                              long long* __restrict__ keep, long long* __restrict__ n_keep) {
  extern __shared__ unsigned long long remv[];
  const long long words = (n + 63) / 64;
  for (long long w = threadIdx.x; w < words; w += blockDim.x) remv[w] = 0ull;
  __syncthreads();
  __shared__ long long s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  for (long long i = 0; i < n; ++i) {
    const bool alive = !((remv[i >> 6] >> (i & 63)) & 1ull);  // uniform: every thread reads the same word
    if (alive) {
      if (threadIdx.x == 0) keep[s_cnt++] = (long long)order[i];
      for (long long w = (i >> 6) + threadIdx.x; w < words; w += blockDim.x) remv[w] |= mask[i * words + w];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *n_keep = s_cnt;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

size_t y5obb_poly_nms_workspace_bytes(int64_t n) {
  if (n <= 0) return 256;
  size_t cub_bytes = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                      (const unsigned int*)nullptr, (unsigned int*)nullptr, (int)n) != cudaSuccess) {
    (void)cudaGetLastError();
    cub_bytes = (size_t)(32u << 20) + (size_t)n * 16;
  }
  const size_t words = (size_t)((n + 63) / 64);
  return 4096 + cub_bytes + (size_t)n * (8 + 8 + 4 + 4) + (size_t)n * words * 8;
}

int y5obb_poly_iou_pairs_f64(const double* p8, const double* q8, double* iou_out, int64_t n, void* stream) {
  if (n < 0) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!p8 || !q8 || !iou_out) return Y5OBB_EINVAL;
  k_poly_pair_iou<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p8, q8, iou_out, n);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_poly_nms_f64(const double* dets9, int64_t n, double thresh, int64_t* keep_out, int64_t* n_keep_out, void* workspace,
                       size_t workspace_bytes, void* stream) {
  if (n < 0 || !keep_out || !n_keep_out) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    Y5_CUDA(cudaMemsetAsync(n_keep_out, 0, sizeof(int64_t), st));
    return Y5OBB_OK;
  }
  if (!dets9 || !workspace || n > 200000) return Y5OBB_EINVAL;  // the dense bit matrix is n^2 / 8 bytes
  if (y5obb_poly_nms_workspace_bytes(n) > workspace_bytes) return Y5OBB_EWORKSPACE;
  const size_t words = (size_t)((n + 63) / 64);
  if (words * 8 > 200 * 1024) return Y5OBB_EINVAL;
  Carver c(workspace);
  unsigned long long* keys_a = c.take<unsigned long long>(n);
  unsigned long long* keys_b = c.take<unsigned long long>(n);
  unsigned int* vals_a = c.take<unsigned int>(n);
  unsigned int* vals_b = c.take<unsigned int>(n);
  unsigned long long* mask = c.take<unsigned long long>((size_t)n * words);
  size_t cub_bytes = workspace_bytes - c.used();
  void* cub_tmp = c.take<char>(1);
  k_poly_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dets9, n, keys_a, vals_a);
  Y5_LAUNCH_CHECK();
  Y5_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, keys_a, keys_b, vals_a, vals_b, (int)n, 0, 64, st));
  const long long total = (long long)n * (long long)words;
  k_poly_mask<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(dets9, vals_b, n, thresh, mask);
  Y5_LAUNCH_CHECK();
  static bool attr = false;
  if (!attr) {
    Y5_CUDA(cudaFuncSetAttribute(k_poly_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  k_poly_reduce<<<1, 1024, words * 8, st>>>(mask, vals_b, n, reinterpret_cast<long long*>(keep_out),
                                            reinterpret_cast<long long*>(n_keep_out));
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
