// Device geometry shared by several kernels:
//   rbox2poly_f32      utils/rboxs_utils.py:106-126 in separately rounded fp32 ops (rbox_utils.cu, scene.cu)
//   py_round           Python's round(x, n) on doubles, exactly (scene.cu, dota_eval.cu)
//   iou_poly_dev       DOTA_devkit/polyiou.cpp:9-128 iou_poly in fp64 without FMA contraction (poly_nms.cu, scene.cu,
//                      dota_eval.cu)
//   poly_suppress_word one 64-column word of the py_cpu_nms_poly_fast suppression matrix (poly_nms.cu, scene.cu)
//   poly_greedy_scan   the greedy keep scan over that matrix by one thread block (poly_nms.cu, scene.cu)
#pragma once
#include "common.cuh"

namespace y5obb {
namespace geom {

__device__ __forceinline__ void rbox2poly_f32(float cx, float cy, float w, float h, float th, float* o) {
  const float c = cosf(th), s = sinf(th);
  const float w2 = __fdiv_rn(w, 2.0f), h2 = __fdiv_rn(h, 2.0f);
  const float v1x = __fmul_rn(w2, c), v1y = __fmul_rn(-w2, s);   // vector1 = (w/2 * Cos, -w/2 * Sin)
  const float v2x = __fmul_rn(-h2, s), v2y = __fmul_rn(-h2, c);  // vector2 = (-h/2 * Sin, -h/2 * Cos)
  o[0] = __fadd_rn(__fadd_rn(cx, v1x), v2x);  // point1 = center + vector1 + vector2
  o[1] = __fadd_rn(__fadd_rn(cy, v1y), v2y);
  o[2] = __fsub_rn(__fadd_rn(cx, v1x), v2x);  // point2 = center + vector1 - vector2
  o[3] = __fsub_rn(__fadd_rn(cy, v1y), v2y);
  o[4] = __fsub_rn(__fsub_rn(cx, v1x), v2x);  // point3 = center - vector1 - vector2
  o[5] = __fsub_rn(__fsub_rn(cy, v1y), v2y);
  o[6] = __fadd_rn(__fsub_rn(cx, v1x), v2x);  // point4 = center - vector1 + vector2
  o[7] = __fadd_rn(__fsub_rn(cy, v1y), v2y);
}

// Python's round(x, n) for p10 = 10^n on a double |x| * p10 < 2^52: the nearest integer to the EXACT product, ties to even
// (py_round_int), divided by 10^n in IEEE arithmetic (the double strtod returns for the rounded decimal string).
// x * p10 = y + e exactly; the correction applies when y is a tie but the exact product is not.
__device__ __forceinline__ double py_round_int(double x, double p10) {
  const double y = __dmul_rn(x, p10);
  const double e = __fma_rn(x, p10, -y);
  double k = rint(y);
  if (fabs(__dsub_rn(y, k)) == 0.5 && e != 0.0) k = e > 0.0 ? __dadd_rn(y, 0.5) : __dsub_rn(y, 0.5);
  return k;
}
__device__ __forceinline__ double py_round(double x, double p10) { return __ddiv_rn(py_round_int(x, p10), p10); }

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
__device__ inline double parea(const P2* ps, int n) {
  double res = 0.0;
  for (int i = 0; i < n; ++i) {
    const int j = (i + 1 == n) ? 0 : i + 1;
    res = padd(res, psub(pmul(ps[i].x, ps[j].y), pmul(ps[i].y, ps[j].x)));
  }
  return res / 2.0;
}
__device__ __forceinline__ bool psame(P2 p, P2 q) { return psig(psub(p.x, q.x)) == 0 && psig(psub(p.y, q.y)) == 0; }

// polyiou.cpp:57-70: the part of polygon p (n points, n <= 8) to the left of a->b, in place
__device__ inline void polygon_cut(P2* p, int& n, P2 a, P2 b) {
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
__device__ inline double tri_intersect(P2 a, P2 b, P2 c, P2 d) {
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

__device__ inline double iou_poly_dev(const double* p8, const double* q8) {
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

// Word w of row i of the py_cpu_nms_poly_fast suppression matrix over n candidates in processing order: bit c set = candidate
// w * 64 + c (> i) is suppressed by i, i.e. !(ovr <= thresh) with ovr the axis-aligned pre-filter (areas with the +1 pixel
// convention, intersection without) replaced by the polygon IoU where it is > 0.  row(j) returns candidate j's 8 coordinates.
template <typename Row>
__device__ inline unsigned long long poly_suppress_word(Row row, long long i, long long w, long long n, double thresh) {
  unsigned long long bits = 0ull;
  if ((w + 1) * 64 <= i + 1) return bits;
  const double* di = row(i);
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
    const double* dj = row(j);
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
  return bits;
}

// The greedy scan over such a matrix by one thread block: thread 0 calls keep(slot, i) for every surviving row i, slot counting
// the survivors; returns their number on thread 0.  remv: (n + 63) / 64 words of dynamic shared memory.
template <typename Keep>
__device__ inline long long poly_greedy_scan(const unsigned long long* __restrict__ mask, long long n,
                                             unsigned long long* remv, Keep keep) {
  const long long words = (n + 63) / 64;
  for (long long w = threadIdx.x; w < words; w += blockDim.x) remv[w] = 0ull;
  __syncthreads();
  long long cnt = 0;
  for (long long i = 0; i < n; ++i) {
    const bool alive = !((remv[i >> 6] >> (i & 63)) & 1ull);  // uniform: every thread reads the same word
    if (alive) {
      if (threadIdx.x == 0) keep(cnt, i);
      ++cnt;
      for (long long w = (i >> 6) + threadIdx.x; w < words; w += blockDim.x) remv[w] |= mask[i * words + w];
    }
    __syncthreads();
  }
  return cnt;
}

}  // namespace geom
}  // namespace y5obb
