// Device geometry shared by several kernels:
//   rbox2poly_f32      utils/rboxs_utils.py:106-126 in separately rounded fp32 ops (rbox_utils.cu, scene.cu)
//   py_round           Python's round(x, n) on doubles, exactly (scene.cu, dota_eval.cu)
//   iou_poly_dev       DOTA_devkit/polyiou.cpp:9-128 iou_poly in fp64 without FMA contraction (poly_nms.cu, scene.cu,
//                      dota_eval.cu)
//   poly_suppress_word one 64-column word of the py_cpu_nms_poly_fast suppression matrix (poly_nms.cu, scene.cu)
//   poly_greedy_scan   the greedy keep scan over that matrix by one thread block (poly_nms.cu, scene.cu)
//   csl_value          one element of gaussian_label_cpu's CSL row (rbox_utils.cu, augment.cu)
//   poly2rbox_dev      poly2rbox of one polygon, cv2.minAreaRect restated (rbox_utils.cu, augment.cu)
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


// gaussian_label_cpu (utils/rboxs_utils.py:9-26), element k of the row for `angle` in degrees, fp64 like numpy:
// exp(-(x_j)^2 / (2 sigma^2)), j = (k + int(nc/2 - angle)) mod nc, x_j = j - nc/2
__device__ __forceinline__ float csl_value(double angle, int k, int nc, double sig) {
  const int index = (int)((double)nc / 2.0 - angle);  // int(): truncation toward zero
  int j = (k + index) % nc;
  if (j < 0) j += nc;
  const double x = (double)j - (double)nc / 2.0;
  return (float)exp(-(x * x) / (2.0 * sig * sig));
}

// poly2rbox (utils/rboxs_utils.py:39-81): the arithmetic of the reference is cv2.minAreaRect on the 4 float32 points
// (opencv-python >= 4.5.4, not vendored).  Published algorithm restated (rotcalipers.cpp): convex hull; the minimum-area
// enclosing rectangle has a side collinear with a hull edge.  One thread per polygon, double precision throughout
// (the long-edge result does not depend on which of cv2's equivalent (w, h, angle) forms is used), then the reference's
// own post-processing verbatim: theta = -angle/180*pi, long-edge swap (+pi/2), wrap to [-pi/2, pi/2) with pi = 3.141592.
__device__ __forceinline__ double p2r_cross3(const double* o, const double* a, const double* b) {
  return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0]);
}

__device__ __forceinline__ void poly2rbox_dev(const float* __restrict__ poly, double* __restrict__ o, int use_pi) {
  const double PI_REF = 3.141592;
  double p[4][2];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    p[k][0] = (double)poly[2 * k];
    p[k][1] = (double)poly[2 * k + 1];
  }
  // sort lexicographically (x, then y), drop duplicates
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3 - a; ++b)
      if (p[b][0] > p[b + 1][0] || (p[b][0] == p[b + 1][0] && p[b][1] > p[b + 1][1])) {
        const double tx = p[b][0], ty = p[b][1];
        p[b][0] = p[b + 1][0];
        p[b][1] = p[b + 1][1];
        p[b + 1][0] = tx;
        p[b + 1][1] = ty;
      }
  int m = 0;
  double q[4][2];
  for (int k = 0; k < 4; ++k)
    if (k == 0 || p[k][0] != p[k - 1][0] || p[k][1] != p[k - 1][1]) {
      q[m][0] = p[k][0];
      q[m][1] = p[k][1];
      ++m;
    }
  double x = q[0][0], y = q[0][1], w = 0.0, h = 0.0, angle = 0.0;
  double hull[8][2];
  int nh = 0;
  if (m >= 3) {  // Andrew's monotone chain
    int lo = 0;
    for (int k = 0; k < m; ++k) {
      while (lo >= 2 && p2r_cross3(hull[lo - 2], hull[lo - 1], q[k]) <= 0) --lo;
      hull[lo][0] = q[k][0];
      hull[lo][1] = q[k][1];
      ++lo;
    }
    int up = lo - 1;  // the last lower point is shared
    const int base = up;
    for (int k = m - 1; k >= 0; --k) {
      while (up - base >= 2 && p2r_cross3(hull[up - 2], hull[up - 1], q[k]) <= 0) --up;
      hull[up][0] = q[k][0];
      hull[up][1] = q[k][1];
      ++up;
    }
    nh = up - 1;  // the last upper point is the first lower point
  }
  if (m >= 3 && nh >= 3) {
    double best = -1.0, bu0 = 1, bu1 = 0, amin = 0, amax = 0, bmin = 0, bmax = 0;
    for (int e = 0; e < nh; ++e) {
      const double ex = hull[(e + 1) % nh][0] - hull[e][0], ey = hull[(e + 1) % nh][1] - hull[e][1];
      const double len = hypot(ex, ey);
      const double u0 = ex / len, u1 = ey / len;
      double a0 = 1e300, a1 = -1e300, b0 = 1e300, b1 = -1e300;
      for (int k = 0; k < nh; ++k) {
        const double a = __dadd_rn(__dmul_rn(hull[k][0], u0), __dmul_rn(hull[k][1], u1));
        const double b = __dadd_rn(__dmul_rn(hull[k][0], -u1), __dmul_rn(hull[k][1], u0));
        a0 = fmin(a0, a);
        a1 = fmax(a1, a);
        b0 = fmin(b0, b);
        b1 = fmax(b1, b);
      }
      const double area = __dmul_rn(a1 - a0, b1 - b0);
      if (best < 0 || area < best * (1 - 1e-12)) {
        best = area;
        bu0 = u0;
        bu1 = u1;
        amin = a0;
        amax = a1;
        bmin = b0;
        bmax = b1;
      }
    }
    const double ca = (amax + amin) / 2, cb = (bmax + bmin) / 2;
    x = __dadd_rn(__dmul_rn(bu0, ca), __dmul_rn(-bu1, cb));
    y = __dadd_rn(__dmul_rn(bu1, ca), __dmul_rn(bu0, cb));
    const double eu = amax - amin, en = bmax - bmin;
    double alpha = fmod(atan2(bu1, bu0) * (180.0 / 3.14159265358979323846), 180.0);
    if (alpha < 0) alpha += 180.0;
    if (alpha < 1e-9 || alpha > 180.0 - 1e-9) {
      w = en;
      h = eu;
      angle = 90.0;
    } else if (alpha <= 90.0) {
      w = eu;
      h = en;
      angle = alpha;
    } else {
      w = en;
      h = eu;
      angle = alpha - 90.0;
    }
  } else if (m == 2 || (m >= 3 && nh == 2)) {  // a segment: its two extreme points are the first and last sorted ones
    const double x0 = q[0][0], y0 = q[0][1], x1 = q[m - 1][0], y1 = q[m - 1][1];
    x = (x0 + x1) / 2;
    y = (y0 + y1) / 2;
    w = hypot(x1 - x0, y1 - y0);
    h = 0.0;
    angle = atan2(y1 - y0, x1 - x0) * (180.0 / 3.14159265358979323846);
  }
  double theta = -angle / 180 * PI_REF;
  if (w != fmax(w, h)) {
    const double t = w;
    w = h;
    h = t;
    theta += PI_REF / 2;
  }
  const double start = -PI_REF / 2;
  double r = fmod(theta - start, PI_REF);  // python %: result has the sign of the divisor
  if (r < 0) r += PI_REF;
  theta = r + start;
  o[0] = x;
  o[1] = y;
  o[2] = w;
  o[3] = h;
  o[4] = use_pi ? theta : theta * 180 / PI_REF + 90;
}

}  // namespace geom
}  // namespace y5obb
