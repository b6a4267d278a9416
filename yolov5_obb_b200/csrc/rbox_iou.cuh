// Rotated-box IoU for sm_90a — device restatement of the reference's *device* code path
//   utils/nms_rotated/src/box_iou_rotated_utils.h:57-360 (the __CUDACC__ branch:
//   exchange-sort hull ordering, :195-218), called per pair by nms_rotated_cuda.cu:57-62.
//
// Parity contract: every floating-point expression below has the same operand order and the same
// float/double mix as the reference expression it restates (cited per block), and this file is
// compiled with nvcc's default -fmad=true like the reference extension.  Which products ptxas fuses
// into FMAs still depends on the surrounding program: on sm_90a 17.9 % of the IoUs of
// tests/test_nms_gpu.py's 400 000 near pairs differ from the reference device function, by at most
// 4 ulp; degenerate pairs and every tested keep list of the reference's CUDA kernel are equal.
//
// What is NOT the reference's design: trig and area are computed once per box (PreBox), not once per
// pair; the caller rejects far-apart pairs before calling this (exact: such pairs have IoU == 0).
#pragma once
#include <cuda_runtime.h>

namespace y5obb {

// Per-box precompute.  c2/s2 = (float)cos/sin((double)theta) * 0.5f  (utils.h:63-65), area = w*h (:349-350)
struct PreBox {
  float cx, cy, w, h;
  float c2, s2, area, rad;  // rad: conservative circumradius used only for the exact far-pair reject
};

struct Pt {
  float x, y;
};

__device__ __forceinline__ float cross2(const Pt& A, const Pt& B) { return A.x * B.y - B.x * A.y; }  // utils.h:52-55
__device__ __forceinline__ float dot2(const Pt& A, const Pt& B) { return A.x * B.x + A.y * B.y; }    // utils.h:45-48
__device__ __forceinline__ Pt psub(const Pt& A, const Pt& B) { return Pt{A.x - B.x, A.y - B.y}; }

// utils.h:66-74 with the centre already shifted
__device__ __forceinline__ void box_corners(float xc, float yc, float w, float h, float c2, float s2, Pt (&p)[4]) {
  p[0].x = xc + s2 * h + c2 * w;
  p[0].y = yc + c2 * h - s2 * w;
  p[1].x = xc - s2 * h + c2 * w;
  p[1].y = yc - c2 * h - s2 * w;
  p[2].x = 2 * xc - p[0].x;
  p[2].y = 2 * yc - p[0].y;
  p[3].x = 2 * xc - p[1].x;
  p[3].y = 2 * yc - p[1].y;
}

// utils.h:77-156
__device__ __forceinline__ int gather_points(const Pt (&r1)[4], const Pt (&r2)[4], Pt (&out)[24]) {
  Pt e1[4], e2[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    e1[i] = psub(r1[(i + 1) % 4], r1[i]);
    e2[i] = psub(r2[(i + 1) % 4], r2[i]);
  }
  int n = 0;
#pragma unroll
  for (int i = 0; i < 4; i++) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float det = cross2(e2[j], e1[i]);
      if (fabs(det) <= 1e-14) continue;  // float promoted to double, as in utils.h:99
      Pt d = psub(r2[j], r1[i]);
      float t1 = cross2(e2[j], d) / det;
      float t2 = cross2(e1[i], d) / det;
      if (t1 >= 0.0f && t1 <= 1.0f && t2 >= 0.0f && t2 <= 1.0f) {
        out[n].x = r1[i].x + e1[i].x * t1;
        out[n].y = r1[i].y + e1[i].y * t1;
        n++;
      }
    }
  }
  {  // corners of r1 inside r2 (utils.h:115-134)
    const Pt& AB = e2[0];
    const Pt& DA = e2[3];
    float ABAB = dot2(AB, AB), ADAD = dot2(DA, DA);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      Pt AP = psub(r1[i], r2[0]);
      float pab = dot2(AP, AB);
      float pad = -dot2(AP, DA);
      if ((pab >= 0) && (pad >= 0) && (pab <= ABAB) && (pad <= ADAD)) out[n++] = r1[i];
    }
  }
  {  // corners of r2 inside r1 (utils.h:137-153)
    const Pt& AB = e1[0];
    const Pt& DA = e1[3];
    float ABAB = dot2(AB, AB), ADAD = dot2(DA, DA);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      Pt AP = psub(r2[i], r1[0]);
      float pab = dot2(AP, AB);
      float pad = -dot2(AP, DA);
      if ((pab >= 0) && (pad >= 0) && (pab <= ABAB) && (pad <= ADAD)) out[n++] = r2[i];
    }
  }
  return n;
}

// utils.h:158-291, device branch, shift_to_zero = true.  Returns hull size; hull in q[0..m).
__device__ __forceinline__ int hull_order(const Pt (&p)[24], int n, Pt (&q)[24]) {
  int t = 0;
  for (int i = 1; i < n; i++)
    if (p[i].y < p[t].y || (p[i].y == p[t].y && p[i].x < p[t].x)) t = i;
  const Pt s = p[t];
  for (int i = 0; i < n; i++) q[i] = psub(p[i], s);
  Pt tmp = q[0];
  q[0] = q[t];
  q[t] = tmp;
  float dist[24];
  for (int i = 0; i < n; i++) dist[i] = dot2(q[i], q[i]);
  for (int i = 1; i < n - 1; i++)
    for (int j = i + 1; j < n; j++) {
      float cp = cross2(q[i], q[j]);
      if ((cp < -1e-6) || (fabs(cp) < 1e-6 && dist[i] > dist[j])) {
        Pt qt = q[i];
        q[i] = q[j];
        q[j] = qt;
        float dt = dist[i];
        dist[i] = dist[j];
        dist[j] = dt;
      }
    }
  int k;
  for (k = 1; k < n; k++)
    if (dist[k] > 1e-8) break;
  if (k == n) {
    q[0] = p[t];
    return 1;
  }
  q[1] = q[k];
  int m = 2;
  for (int i = k + 1; i < n; i++) {
    while (m > 1) {
      Pt a = psub(q[i], q[m - 2]), b = psub(q[m - 1], q[m - 2]);
      // two separately rounded products compared, never a fused difference (utils.h:262-270)
      if (__fmul_rn(a.x, b.y) >= __fmul_rn(b.x, a.y))
        m--;
      else
        break;
    }
    q[m++] = q[i];
  }
  return m;
}

// utils.h:293-305
__device__ __forceinline__ float hull_area(const Pt (&q)[24], int m) {
  if (m <= 2) return 0;
  float area = 0;
  for (int i = 1; i < m - 1; i++) area += fabs(cross2(psub(q[i], q[0]), psub(q[i + 1], q[0])));
  return area / 2.0;
}

// utils.h:334-360.  A and B in the caller's (unshifted) coordinates.
__device__ __noinline__ float rbox_iou(const PreBox& A, const PreBox& B) {
  auto sx = (A.cx + B.cx) / 2.0;  // float add, double divide (utils.h:338-339)
  auto sy = (A.cy + B.cy) / 2.0;
  float ax = A.cx - sx, ay = A.cy - sy;  // double subtract, rounded to float on store (:340-341,:345-346)
  float bx = B.cx - sx, by = B.cy - sy;
  if (A.area < 1e-14 || B.area < 1e-14) return 0.f;
  Pt ra[4], rb[4], cand[24], ord[24];
  box_corners(ax, ay, A.w, A.h, A.c2, A.s2, ra);
  box_corners(bx, by, B.w, B.h, B.c2, B.s2, rb);
  int n = gather_points(ra, rb, cand);
  float inter;
  if (n <= 2) {
    inter = 0.0;
  } else {
    int m = hull_order(cand, n, ord);
    inter = hull_area(ord, m);
  }
  return inter / (A.area + B.area - inter);
}

__device__ __forceinline__ PreBox make_prebox(float cx, float cy, float w, float h, float a) {
  PreBox b;
  b.cx = cx;
  b.cy = cy;
  b.w = w;
  b.h = h;
  double th = a;
  b.c2 = (float)cos(th) * 0.5f;
  b.s2 = (float)sin(th) * 0.5f;
  b.area = w * h;
  // circumradius, inflated: any pair with centre distance beyond the radius sum has no contact in the
  // reference arithmetic either (its error is ~1e-7 relative), hence IoU == 0 exactly
  b.rad = 0.5f * sqrtf(w * w + h * h) * 1.001f + 1e-3f;
  return b;
}

}  // namespace y5obb
