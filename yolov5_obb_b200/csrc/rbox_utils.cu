// Post-NMS geometry and CSL targets (HBM-bound elementwise kernels; one thread per box):
//   y5obb_rbox2poly_f32      utils/rboxs_utils.py:106-126  (torch branch of rbox2poly)
//   y5obb_poly2hbb_f32       utils/rboxs_utils.py:147-165  (torch branch of poly2hbb)
//   y5obb_scale_polys_f32    utils/general.py:636-650      (scale_polys, in place)
//   y5obb_scale_polys_batched_f32  both of the above for a batch's packed NMS rows, one (pad, gain) per image
//   y5obb_gaussian_label     utils/rboxs_utils.py:9-26     (gaussian_label_cpu: 180-bin CSL row)
// Each arithmetic step is a separately rounded fp32 op (no FMA contraction), like the chain of ATen
// elementwise kernels it replaces; the CSL row is evaluated in fp64 like the numpy original.
#include <algorithm>

#include "common.cuh"
#include "geom.cuh"

namespace y5obb {
namespace {

__global__ void k_rbox2poly(const float* __restrict__ r, float* __restrict__ p, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  geom::rbox2poly_f32(r[5 * i], r[5 * i + 1], r[5 * i + 2], r[5 * i + 3], r[5 * i + 4], p + 8 * i);
}

__global__ void k_poly2hbb(const float* __restrict__ p, float* __restrict__ hbb, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* q = p + 8 * i;
  const float xmax = fmaxf(fmaxf(q[0], q[2]), fmaxf(q[4], q[6])), xmin = fminf(fminf(q[0], q[2]), fminf(q[4], q[6]));
  const float ymax = fmaxf(fmaxf(q[1], q[3]), fmaxf(q[5], q[7])), ymin = fminf(fminf(q[1], q[3]), fminf(q[5], q[7]));
  hbb[4 * i] = __fdiv_rn(__fadd_rn(xmax, xmin), 2.0f);
  hbb[4 * i + 1] = __fdiv_rn(__fadd_rn(ymax, ymin), 2.0f);
  hbb[4 * i + 2] = __fsub_rn(xmax, xmin);
  hbb[4 * i + 3] = __fsub_rn(ymax, ymin);
}

__global__ void k_scale_polys(float* __restrict__ p, int64_t n, float padx, float pady, float gain) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 8) return;
  const float pad = (i & 1) ? pady : padx;
  p[i] = __fdiv_rn(__fsub_rn(p[i], pad), gain);
}

__global__ void k_scale_polys_batched(const float* __restrict__ rows7, const int64_t* __restrict__ counts,
                                      const float* __restrict__ pg, int B, int max_det, float* __restrict__ polys) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)B * max_det) return;
  const int b = (int)(i / max_det);
  float poly[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (i - (int64_t)b * max_det < counts[b]) {
    const float* r = rows7 + i * 7;
    geom::rbox2poly_f32(r[0], r[1], r[2], r[3], r[4], poly);
    const float gain = pg[3 * b + 2];
#pragma unroll
    for (int k = 0; k < 8; ++k) poly[k] = __fdiv_rn(__fsub_rn(poly[k], pg[3 * b + (k & 1)]), gain);
  }
  float4* o = reinterpret_cast<float4*>(polys + i * 8);
  o[0] = make_float4(poly[0], poly[1], poly[2], poly[3]);
  o[1] = make_float4(poly[4], poly[5], poly[6], poly[7]);
}

__global__ void k_gaussian_label(const double* __restrict__ angle, float* __restrict__ out, int64_t n, int nc, double sig) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * nc) return;
  const int64_t row = i / nc;
  out[i] = geom::csl_value(angle[row], (int)(i - row * nc), nc, sig);
}

__global__ void k_poly2rbox(const float* __restrict__ polys, double* __restrict__ out, long long n, int use_pi) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  geom::poly2rbox_dev(polys + i * 8, out + i * 5, use_pi);
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_rbox2poly_f32(const float* rboxes5, float* polys8, int64_t n, void* stream) {
  if (n < 0) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!rboxes5 || !polys8) return Y5OBB_EINVAL;
  k_rbox2poly<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rboxes5, polys8, n);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_poly2hbb_f32(const float* polys8, float* hbb4, int64_t n, void* stream) {
  if (n < 0) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!polys8 || !hbb4) return Y5OBB_EINVAL;
  k_poly2hbb<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(polys8, hbb4, n);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_scale_polys_f32(float* polys8, int64_t n, float pad_x, float pad_y, float gain, void* stream) {
  if (n < 0 || gain == 0.0f) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!polys8) return Y5OBB_EINVAL;
  k_scale_polys<<<(unsigned)((n * 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(polys8, n, pad_x, pad_y, gain);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_scale_polys_batched_f32(const float* rows7, const int64_t* counts, const float* pad_gain3, int B, int max_det,
                                  float* polys8, void* stream) {
  if (B < 0 || max_det < 0) return Y5OBB_EINVAL;
  if (B == 0 || max_det == 0) return Y5OBB_OK;
  if (!rows7 || !counts || !pad_gain3 || !polys8 || (reinterpret_cast<uintptr_t>(polys8) & 15)) return Y5OBB_EINVAL;
  const int64_t n = (int64_t)B * max_det;
  k_scale_polys_batched<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rows7, counts, pad_gain3, B, max_det,
                                                                                    polys8);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_poly2rbox(const float* polys8, double* rbox5, int64_t n, int use_pi, void* stream) {
  if (n < 0) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!polys8 || !rbox5) return Y5OBB_EINVAL;
  k_poly2rbox<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(polys8, rbox5, n, use_pi);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_gaussian_label(const double* angle_deg, float* csl_out, int64_t n, int num_class, double sigma, void* stream) {
  if (n < 0 || num_class <= 0 || !(sigma > 0)) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!angle_deg || !csl_out) return Y5OBB_EINVAL;
  k_gaussian_label<<<(unsigned)((n * num_class + 255) / 256), 256, 0, (cudaStream_t)stream>>>(angle_deg, csl_out, n,
                                                                                              num_class, sigma);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
