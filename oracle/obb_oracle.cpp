// CPU oracle for the rotated-box path (TEST INFRASTRUCTURE — never linked into the product library).
//
// Restates, in scalar C++ with no FMA contraction (build with -ffp-contract=off), the algorithm of
//   utils/nms_rotated/src/box_iou_rotated_utils.h:57-360   (single_box_iou_rotated)
//   utils/nms_rotated/src/nms_rotated_cpu.cpp:8-61          (greedy NMS, suppress if IoU >= thr)
//   utils/nms_rotated/src/nms_rotated_cuda.cu:12-134        (greedy NMS, suppress if IoU >  thr)
//   utils/nms_rotated/nms_rotated_wrapper.py:6-46           (min(w,h) < 0.001 pre-filter)
//   utils/general.py:772-862                                (non_max_suppression_obb)
//
// Two hull-ordering variants exist in the reference and both are restated here:
//   variant 0 ("host"):   std::sort with the angle/distance comparator (box_iou_rotated_utils.h:221-233)
//   variant 1 ("device"): the O(n^2) exchange sort used under __CUDACC__   (box_iou_rotated_utils.h:195-218)
// Variant 1 reproduces the device ORDER of operations but not nvcc's FMA contraction; the GPU tests
// therefore compare IoU values against it with a tolerance and keep lists on inputs whose decisive
// IoUs are not within that tolerance of the threshold; bit-for-bit device parity is checked against
// oracle/_ref (the reference's own kernels compiled by oracle/build_ref.py).
//
// Pinning: oracle/_ref/nms_rotated_ref (reference CPU extension built here) must agree with variant 0
// bit for bit — tests/test_oracle_pin.py and the committed tests/golden/*.npz check exactly that.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <numeric>
#include <vector>

namespace {

struct P2 {
  float x, y;
};

inline float cross2(const P2& a, const P2& b) { return a.x * b.y - b.x * a.y; }
inline float dot2(const P2& a, const P2& b) { return a.x * b.x + a.y * b.y; }
inline P2 sub(const P2& a, const P2& b) { return P2{a.x - b.x, a.y - b.y}; }

struct RBox {
  float cx, cy, w, h, a;
};

// box_iou_rotated_utils.h:57-75 — trig in double, cast to float, then * 0.5f
void corners(const RBox& b, P2 (&p)[4]) {
  double th = b.a;
  float c2 = (float)std::cos(th) * 0.5f;
  float s2 = (float)std::sin(th) * 0.5f;
  p[0].x = b.cx + s2 * b.h + c2 * b.w;
  p[0].y = b.cy + c2 * b.h - s2 * b.w;
  p[1].x = b.cx - s2 * b.h + c2 * b.w;
  p[1].y = b.cy - c2 * b.h - s2 * b.w;
  p[2].x = 2 * b.cx - p[0].x;
  p[2].y = 2 * b.cy - p[0].y;
  p[3].x = 2 * b.cx - p[1].x;
  p[3].y = 2 * b.cy - p[1].y;
}

// box_iou_rotated_utils.h:77-156
int candidate_points(const P2 (&r1)[4], const P2 (&r2)[4], P2 (&out)[24]) {
  P2 e1[4], e2[4];
  for (int i = 0; i < 4; ++i) {
    e1[i] = sub(r1[(i + 1) & 3], r1[i]);
    e2[i] = sub(r2[(i + 1) & 3], r2[i]);
  }
  int n = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      float det = cross2(e2[j], e1[i]);
      if (std::fabs(det) <= 1e-14) continue;  // parallel edges (double compare)
      P2 d = sub(r2[j], r1[i]);
      float t1 = cross2(e2[j], d) / det;
      float t2 = cross2(e1[i], d) / det;
      if (t1 >= 0.0f && t1 <= 1.0f && t2 >= 0.0f && t2 <= 1.0f)
        out[n++] = P2{r1[i].x + e1[i].x * t1, r1[i].y + e1[i].y * t1};
    }
  // corners of r1 inside r2, then corners of r2 inside r1
  for (int pass = 0; pass < 2; ++pass) {
    const P2(&in)[4] = pass == 0 ? r1 : r2;
    const P2(&rect)[4] = pass == 0 ? r2 : r1;
    const P2(&e)[4] = pass == 0 ? e2 : e1;
    const P2& AB = e[0];
    const P2& DA = e[3];
    float ABAB = dot2(AB, AB), ADAD = dot2(DA, DA);
    for (int i = 0; i < 4; ++i) {
      P2 AP = sub(in[i], rect[0]);
      float pab = dot2(AP, AB);
      float pad = -dot2(AP, DA);
      if (pab >= 0 && pad >= 0 && pab <= ABAB && pad <= ADAD) out[n++] = in[i];
    }
  }
  return n;
}

// box_iou_rotated_utils.h:158-291 (shift_to_zero = true: only the area is wanted)
int hull(const P2 (&p)[24], int n, P2 (&q)[24], int variant) {
  int t = 0;
  for (int i = 1; i < n; ++i)
    if (p[i].y < p[t].y || (p[i].y == p[t].y && p[i].x < p[t].x)) t = i;
  const P2 s = p[t];
  for (int i = 0; i < n; ++i) q[i] = sub(p[i], s);
  std::swap(q[0], q[t]);
  float dist[24];
  if (variant == 1) {
    for (int i = 0; i < n; ++i) dist[i] = dot2(q[i], q[i]);
    for (int i = 1; i < n - 1; ++i)
      for (int j = i + 1; j < n; ++j) {
        float cp = cross2(q[i], q[j]);
        if ((cp < -1e-6) || (std::fabs(cp) < 1e-6 && dist[i] > dist[j])) {
          std::swap(q[i], q[j]);
          std::swap(dist[i], dist[j]);
        }
      }
  } else {
    std::sort(q + 1, q + n, [](const P2& A, const P2& B) -> bool {
      float c = cross2(A, B);
      if (std::fabs(c) < 1e-6) return dot2(A, A) < dot2(B, B);
      return c > 0;
    });
    for (int i = 0; i < n; ++i) dist[i] = dot2(q[i], q[i]);
  }
  int k = 1;
  while (k < n && !(dist[k] > 1e-8)) ++k;
  if (k == n) {
    q[0] = p[t];
    return 1;
  }
  q[1] = q[k];
  int m = 2;
  for (int i = k + 1; i < n; ++i) {
    while (m > 1) {
      P2 a = sub(q[i], q[m - 2]), b = sub(q[m - 1], q[m - 2]);
      if (a.x * b.y >= b.x * a.y)
        --m;
      else
        break;
    }
    q[m++] = q[i];
  }
  return m;
}

// box_iou_rotated_utils.h:293-305
float fan_area(const P2 (&q)[24], int m) {
  if (m <= 2) return 0;
  float area = 0;
  for (int i = 1; i < m - 1; ++i) area += std::fabs(cross2(sub(q[i], q[0]), sub(q[i + 1], q[0])));
  return (float)(area / 2.0);
}

// box_iou_rotated_utils.h:334-360
float iou_rotated(const float* a, const float* b, int variant) {
  double sx = (a[0] + b[0]) / 2.0;
  double sy = (a[1] + b[1]) / 2.0;
  RBox A{(float)(a[0] - sx), (float)(a[1] - sy), a[2], a[3], a[4]};
  RBox B{(float)(b[0] - sx), (float)(b[1] - sy), b[2], b[3], b[4]};
  float areaA = A.w * A.h, areaB = B.w * B.h;
  if (areaA < 1e-14 || areaB < 1e-14) return 0.f;
  P2 ra[4], rb[4], cand[24], ord[24];
  corners(A, ra);
  corners(B, rb);
  int n = candidate_points(ra, rb, cand);
  float inter = 0.f;
  if (n > 2) {
    int m = hull(cand, n, ord, variant);
    inter = fan_area(ord, m);
  }
  return inter / (areaA + areaB - inter);
}

}  // namespace

extern "C" {

// IoU of n independent pairs a[i], b[i] (5 floats each).
void oracle_iou_pairs(const float* a, const float* b, float* out, int64_t n, int variant) {
  for (int64_t i = 0; i < n; ++i) out[i] = iou_rotated(a + 5 * i, b + 5 * i, variant);
}

// Greedy rotated NMS.  mode 0 = reference CPU semantics (suppress if IoU >= thr, host hull),
// mode 1 = reference CUDA semantics (suppress if IoU > thr, device hull order).
// Order: descending score, ties by ascending index (the reference's sort is unstable; tests use
// unique scores).  keep[] receives indices into the caller's arrays; returns the count.
int64_t oracle_nms_rotated(const float* dets, const float* scores, int64_t n, float thr, int mode,
                           int64_t* keep) {
  std::vector<int64_t> order(n);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int64_t x, int64_t y) { return scores[x] > scores[y]; });
  std::vector<uint8_t> dead(n, 0);
  int64_t nk = 0;
  for (int64_t ii = 0; ii < n; ++ii) {
    int64_t i = order[ii];
    if (dead[i]) continue;
    keep[nk++] = i;
    for (int64_t jj = ii + 1; jj < n; ++jj) {
      int64_t j = order[jj];
      if (dead[j]) continue;
      float v = iou_rotated(dets + 5 * i, dets + 5 * j, mode);
      if (mode == 0 ? (v >= thr) : (v > thr)) dead[j] = 1;
    }
  }
  return nk;
}

// obb_nms wrapper semantics (nms_rotated_wrapper.py:26-42): boxes with min(w,h) < 0.001 never enter
// NMS and are never returned.
int64_t oracle_obb_nms(const float* dets, const float* scores, int64_t n, float thr, int mode, int64_t* keep) {
  std::vector<int64_t> ori;
  std::vector<float> d, s;
  for (int64_t i = 0; i < n; ++i) {
    float mn = std::min(dets[5 * i + 2], dets[5 * i + 3]);
    if (!(mn < 0.001f)) {
      ori.push_back(i);
      d.insert(d.end(), dets + 5 * i, dets + 5 * i + 5);
      s.push_back(scores[i]);
    }
  }
  if (ori.empty()) return 0;
  std::vector<int64_t> k(ori.size());
  int64_t nk = oracle_nms_rotated(d.data(), s.data(), (int64_t)ori.size(), thr, mode, k.data());
  for (int64_t i = 0; i < nk; ++i) keep[i] = ori[k[i]];
  return nk;
}

}  // extern "C"
