// Training augmentation of a batch (utils/datasets.py:561-672 and utils/augmentations.py), from per-sample host plans
// (yolov5_obb_b200/augment.py):
//   y5obb_augment_images_u8   one thread per output pixel: the virtual mosaic / letterbox canvas, cv2.warpAffine's fixed
//                             point bilinear warp, mixup, augment_hsv's cvtColor round trip with LUTs, flips, BGR -> RGB
//   y5obb_augment_labels      one thread per source label: pads, poly_filter, xy @ M.T, flips, poly2rbox, labels_mask;
//                             one scan compacts the survivors in (sample, label) order into collate_fn's rows
// Every step is written with separately rounded operations (no FMA contraction) unless the host arithmetic it restates
// fuses them; the comments name those places.
#include <cub/cub.cuh>

#include "common.cuh"
#include "geom.cuh"

namespace y5obb {
namespace {

constexpr int BORDER = 114;
constexpr int AB_BITS = 10, INTER_BITS = 5;

struct ImgMeta {  // one row of the dataset's [n, 5] int64 table
  int64_t off, h, w, loff, nlab;
};

__device__ __forceinline__ ImgMeta meta_of(const int64_t* m, int id) {
  const int64_t* r = m + 5 * (int64_t)id;
  return ImgMeta{r[0], r[1], r[2], r[3], r[4]};
}

// One channel triple of the canvas of group g at (cx, cy): the placed image whose rectangle holds the point, else 114.
__device__ __forceinline__ void canvas_px(const uint8_t* __restrict__ images, const int64_t* __restrict__ meta,
                                          int n_images, const y5obb_augment_sample& r, int g, int cx, int cy, int* px) {
  px[0] = px[1] = px[2] = BORDER;
  const int side = r.canvas[g];
  if (cx < 0 || cy < 0 || cx >= side || cy >= side) return;
  for (int i = 0; i < r.n_place[g]; ++i) {
    const int p = 4 * g + i;
    const int* q = r.rect + 4 * p;
    if (cx >= q[0] && cx < q[2] && cy >= q[1] && cy < q[3]) {
      const int id = r.img[p];
      if (id < 0 || id >= n_images) return;
      const ImgMeta mi = meta_of(meta, id);
      const int sx = cx - r.pad[2 * p], sy = cy - r.pad[2 * p + 1];
      if (sx < 0 || sy < 0 || sx >= mi.w || sy >= mi.h) return;
      const uint8_t* s = images + mi.off + 3 * ((int64_t)sy * mi.w + sx);
      px[0] = s[0];
      px[1] = s[1];
      px[2] = s[2];
      return;
    }
  }
}

// cv2.warpAffine, INTER_LINEAR, BORDER_CONSTANT 114, for the output pixel (x, y): X = (X0 + adelta[x]) >> 5 with
// adelta[x] = rint(m0 x 1024), X0 = rint((m1 y + m2) 1024) + 16; weights of the 32 x 32 table (exact: products of 1/32
// steps times 2^15), result (sum + 2^14) >> 15.
__device__ __forceinline__ void warp_px(const uint8_t* __restrict__ images, const int64_t* __restrict__ meta, int n_images,
                                        const y5obb_augment_sample& r, int g, int x, int y, int* out) {
  const double* m = r.minv + 6 * g;
  const double sc = (double)(1 << AB_BITS);
  const int rd = (1 << AB_BITS) >> INTER_BITS >> 1;
  const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)x), sc));
  const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)x), sc));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), sc)) + rd;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), sc)) + rd;
  const int X = (X0 + adelta) >> (AB_BITS - INTER_BITS), Y = (Y0 + bdelta) >> (AB_BITS - INTER_BITS);
  const int ix = X >> INTER_BITS, iy = Y >> INTER_BITS, fx = X & 31, fy = Y & 31;
  int acc[3] = {0, 0, 0};
#pragma unroll
  for (int dy = 0; dy < 2; ++dy)
#pragma unroll
    for (int dx = 0; dx < 2; ++dx) {
      const int w = (dy ? fy : 32 - fy) * (dx ? fx : 32 - fx) * 32;
      int px[3];
      canvas_px(images, meta, n_images, r, g, ix + dx, iy + dy, px);
      acc[0] += w * px[0];
      acc[1] += w * px[1];
      acc[2] += w * px[2];
    }
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c] = (acc[c] + (1 << 14)) >> 15;
}

// cv2.COLOR_BGR2HSV, 8U: 12-bit tables sdiv[i] = rint((255 << 12) / i), hdiv[i] = rint((180 << 12) / (6 i)).
__device__ __forceinline__ void bgr2hsv(const int* bgr, int* hsv) {
  const int b = bgr[0], g = bgr[1], r = bgr[2];
  const int v = max(max(b, g), r), vmin = min(min(b, g), r), diff = v - vmin;
  const int sdiv = v ? __double2int_rn(__ddiv_rn((double)(255 << 12), (double)v)) : 0;
  const int hdiv = diff ? __double2int_rn(__ddiv_rn((double)(180 << 12), __dmul_rn(6.0, (double)diff))) : 0;
  const int s = (diff * sdiv + (1 << 11)) >> 12;
  int h = v == r ? g - b : (v == g ? b - r + 2 * diff : r - g + 4 * diff);
  h = (h * hdiv + (1 << 11)) >> 12;
  if (h < 0) h += 180;
  hsv[0] = h;
  hsv[1] = s;
  hsv[2] = v;
}

// cv2.COLOR_HSV2BGR, 8U, as OpenCV 4.13's vector loop computes it (whole blocks of 4 SIMD widths of a row; S % 32 == 0
// keeps every pixel in such blocks with 8-lane vectors): fp32 sector formula with 1 - s*f as one fused multiply-add, then
// trunc(x * 255).
__device__ __forceinline__ void hsv2bgr(const int* hsv, int* bgr) {
  float h = __fmul_rn((float)hsv[0], 6.0f / 180.0f);
  const float sec_f = floorf(h);
  const float f = __fsub_rn(h, sec_f);
  int sec = (int)sec_f % 6;
  const float s = __fmul_rn((float)hsv[1], 1.0f / 255.0f), v = __fmul_rn((float)hsv[2], 1.0f / 255.0f);
  float tab[4];
  tab[0] = v;
  tab[1] = __fmul_rn(v, __fsub_rn(1.0f, s));
  tab[2] = __fmul_rn(v, __fmaf_rn(-s, f, 1.0f));
  tab[3] = __fmul_rn(v, __fmaf_rn(-s, __fsub_rn(1.0f, f), 1.0f));
  const int sd[6][3] = {{1, 3, 0}, {1, 0, 2}, {3, 0, 1}, {0, 2, 1}, {0, 1, 3}, {2, 1, 0}};
#pragma unroll
  for (int c = 0; c < 3; ++c) bgr[c] = min(255, max(0, __float2int_rz(__fmul_rn(tab[sd[sec][c]], 255.0f))));
}

__global__ void k_augment_images(const uint8_t* __restrict__ images, const int64_t* __restrict__ meta, int n_images,
                                 const y5obb_augment_sample* __restrict__ recs, int S, uint8_t* __restrict__ out) {
  const int b = blockIdx.z;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= S || y >= S) return;
  const y5obb_augment_sample& r = recs[b];
  // the flips come last in __getitem__: output (x, y) shows the augmented image at (sx, sy)
  const int sx = (r.flags & Y5OBB_AUG_FLIPLR) ? S - 1 - x : x;
  const int sy = (r.flags & Y5OBB_AUG_FLIPUD) ? S - 1 - y : y;
  int px[3];
  warp_px(images, meta, n_images, r, 0, sx, sy, px);
  if (r.flags & Y5OBB_AUG_MIXUP) {  // (im * r + im2 * (1 - r)).astype(np.uint8): fp64, truncation
    int p2[3];
    warp_px(images, meta, n_images, r, 1, sx, sy, p2);
#pragma unroll
    for (int c = 0; c < 3; ++c)
      px[c] = (int)__dadd_rn(__dmul_rn((double)px[c], r.mix_r), __dmul_rn((double)p2[c], r.mix_1mr));
  }
  if (r.flags & Y5OBB_AUG_HSV) {
    int hsv[3];
    bgr2hsv(px, hsv);
#pragma unroll
    for (int c = 0; c < 3; ++c) hsv[c] = r.lut[256 * c + hsv[c]];
    hsv2bgr(hsv, px);
  }
  const int64_t plane = (int64_t)S * S;
  uint8_t* o = out + (int64_t)b * 3 * plane + (int64_t)y * S + x;
  o[0] = (uint8_t)px[2];  // RGB planes from BGR pixels
  o[plane] = (uint8_t)px[1];
  o[2 * plane] = (uint8_t)px[0];
}

// poly_filter (utils/rboxs_utils.py:183-199) on fp32 or fp64 points: the centre of the axis-aligned hull inside (0, side)
template <typename T>
__device__ __forceinline__ bool poly_keep(const T* q, T side);
template <>
__device__ __forceinline__ bool poly_keep<float>(const float* q, float side) {
  const float xmax = fmaxf(fmaxf(q[0], q[2]), fmaxf(q[4], q[6])), xmin = fminf(fminf(q[0], q[2]), fminf(q[4], q[6]));
  const float ymax = fmaxf(fmaxf(q[1], q[3]), fmaxf(q[5], q[7])), ymin = fminf(fminf(q[1], q[3]), fminf(q[5], q[7]));
  const float xc = __fdiv_rn(__fadd_rn(xmax, xmin), 2.0f), yc = __fdiv_rn(__fadd_rn(ymax, ymin), 2.0f);
  return xc > 0.0f && xc < side && yc > 0.0f && yc < side;
}
template <>
__device__ __forceinline__ bool poly_keep<double>(const double* q, double side) {
  const double xmax = fmax(fmax(q[0], q[2]), fmax(q[4], q[6])), xmin = fmin(fmin(q[0], q[2]), fmin(q[4], q[6]));
  const double ymax = fmax(fmax(q[1], q[3]), fmax(q[5], q[7])), ymin = fmin(fmin(q[1], q[3]), fmin(q[5], q[7]));
  const double xc = __ddiv_rn(__dadd_rn(xmax, xmin), 2.0), yc = __ddiv_rn(__dadd_rn(ymax, ymin), 2.0);
  return xc > 0.0 && xc < side && yc > 0.0 && yc < side;
}

struct LabelOut {  // one candidate's result, in the workspace
  double rb[5];
  float cls;
  int sample;
};

__global__ void k_augment_labels(const float* __restrict__ labels, const int64_t* __restrict__ meta, int n_images,
                                 const y5obb_augment_sample* __restrict__ recs, const int64_t* __restrict__ cand_start,
                                 int B, int64_t ncand, int S, LabelOut* __restrict__ lo, int* __restrict__ keep) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ncand) return;
  int a = 0, z = B * Y5OBB_AUG_MAX_PLACE;  // the slot q with cand_start[q] <= t < cand_start[q + 1]
  while (z - a > 1) {
    const int mid = (a + z) >> 1;
    if (cand_start[mid] <= t) a = mid; else z = mid;
  }
  const int b = a / Y5OBB_AUG_MAX_PLACE, p = a % Y5OBB_AUG_MAX_PLACE, g = p / 4;
  const y5obb_augment_sample& r = recs[b];
  keep[t] = 0;
  const int id = r.img[p];
  if (id < 0 || id >= n_images) return;
  const ImgMeta mi = meta_of(meta, id);
  const int64_t j = t - cand_start[a];
  if (j >= mi.nlab) return;
  const float* L = labels + 9 * (mi.loff + j);
  float q[8];
  const float lw = r.lpad[2 * p], lh = r.lpad[2 * p + 1];
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // labels[:, x] = img_label[:, x] + padw (fp32)
    q[2 * k] = __fadd_rn(L[1 + 2 * k], lw);
    q[2 * k + 1] = __fadd_rn(L[2 + 2 * k], lh);
  }
  const int side = r.canvas[g];
  if (side != S && !poly_keep<float>(q, (float)side)) return;  // load_mosaic's filter on the 2S canvas
  // xy @ M.T in fp64: numpy's matmul goes through BLAS dgemm, whose kernel accumulates x*m0, then y*m1 with a fused
  // multiply-add, then the homogeneous 1*m2
  const double* m = r.m + 6 * g;
  double xy[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double x = q[2 * k], y = q[2 * k + 1];
    xy[2 * k] = __dadd_rn(__fma_rn(y, m[1], __dmul_rn(x, m[0])), m[2]);
    xy[2 * k + 1] = __dadd_rn(__fma_rn(y, m[4], __dmul_rn(x, m[3])), m[5]);
  }
  if (!poly_keep<double>(xy, (double)S)) return;
#pragma unroll
  for (int k = 0; k < 8; ++k) q[k] = (float)xy[k];
  const float fS = (float)S;
  if (r.flags & Y5OBB_AUG_FLIPUD)  // img_h - y - 1: two fp32 roundings
#pragma unroll
    for (int k = 0; k < 4; ++k) q[2 * k + 1] = __fsub_rn(__fsub_rn(fS, q[2 * k + 1]), 1.0f);
  if (r.flags & Y5OBB_AUG_FLIPLR)
#pragma unroll
    for (int k = 0; k < 4; ++k) q[2 * k] = __fsub_rn(__fsub_rn(fS, q[2 * k]), 1.0f);
  LabelOut o;
  geom::poly2rbox_dev(q, o.rb, 1);
  o.cls = L[0];
  o.sample = b;
  lo[t] = o;
  // labels_mask (utils/datasets.py:644-646) as written: (A & B & C & D & E) | F, with cx < img.shape[0] as the 4th term
  const double dS = (double)S;
  keep[t] = ((o.rb[0] >= 0 && o.rb[0] < dS && o.rb[1] >= 0 && o.rb[0] < dS && o.rb[2] > 5) || o.rb[3] > 5) ? 1 : 0;
}

// collate_fn's rows: (image index, cls, cx, cy, l, s, theta, CSL row) as fp32, or compact (.., theta, int(90 - angle))
__global__ void k_augment_rows(const LabelOut* __restrict__ lo, const int* __restrict__ keep,
                               const int* __restrict__ pos, int64_t ncand, int nc, double sig, int tcols,
                               float* __restrict__ rows, int64_t* __restrict__ nt) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t == ncand - 1) *nt = pos[t];
  if (t >= ncand || !keep[t]) return;
  const LabelOut o = lo[t];
  float* row = rows + (int64_t)(pos[t] - 1) * tcols;
  row[0] = (float)o.sample;
  row[1] = o.cls;
#pragma unroll
  for (int k = 0; k < 5; ++k) row[2 + k] = (float)o.rb[k];
  const double angle = o.rb[4] * 180 / 3.141592 + 90;  // utils/rboxs_utils.py:70
  if (tcols == 8) {
    row[7] = (float)trunc((double)nc / 2 - angle);
    return;
  }
  for (int k = 0; k < nc; ++k) row[7 + k] = geom::csl_value(angle, k, nc, sig);
}

size_t labels_ws(int64_t ncand, size_t* scan_bytes) {
  size_t sb = 0;
  cub::DeviceScan::InclusiveSum(nullptr, sb, (const int*)nullptr, (int*)nullptr, (int)(ncand > 0 ? ncand : 1));
  if (scan_bytes) *scan_bytes = sb;
  return align_up(ncand * sizeof(LabelOut), 256) + 2 * align_up(ncand * sizeof(int), 256) + align_up(sb, 256) + 256;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_augment_check(const int64_t* meta, int n_images, int64_t images_bytes, int64_t n_labels,
                        const y5obb_augment_sample* recs, int B, int S) {
  if (n_images <= 0 || B <= 0 || S <= 0 || S % 32 || !meta || !recs || images_bytes < 0 || n_labels < 0)
    return Y5OBB_EINVAL;
  for (int i = 0; i < n_images; ++i) {
    const int64_t* m = meta + 5 * (int64_t)i;
    if (m[1] <= 0 || m[2] <= 0 || m[1] > S || m[2] > S) return Y5OBB_EINVAL;  // images over img_size
    if (m[0] < 0 || m[0] + 3 * m[1] * m[2] > images_bytes) return Y5OBB_EINVAL;
    if (m[3] < 0 || m[4] < 0 || m[3] + m[4] > n_labels) return Y5OBB_EINVAL;
  }
  for (int b = 0; b < B; ++b) {
    const y5obb_augment_sample& r = recs[b];
    const int ng = (r.flags & Y5OBB_AUG_MIXUP) ? 2 : 1;
    for (int g = 0; g < 2; ++g) {
      if (g >= ng) continue;
      const bool mosaic = r.flags & Y5OBB_AUG_MOSAIC;
      if (r.n_place[g] != (mosaic ? 4 : 1) || r.canvas[g] != (mosaic ? 2 * S : S)) return Y5OBB_EINVAL;
      for (int i = 0; i < r.n_place[g]; ++i) {
        const int p = 4 * g + i;
        if (r.img[p] < 0 || r.img[p] >= n_images) return Y5OBB_EINVAL;
        const int64_t* m = meta + 5 * (int64_t)r.img[p];
        const int* q = r.rect + 4 * p;
        if (q[0] < 0 || q[1] < 0 || q[2] > r.canvas[g] || q[3] > r.canvas[g] || q[0] > q[2] || q[1] > q[3]) return Y5OBB_EINVAL;
        const int x0 = q[0] - r.pad[2 * p], y0 = q[1] - r.pad[2 * p + 1];
        const int x1 = q[2] - r.pad[2 * p], y1 = q[3] - r.pad[2 * p + 1];
        if (q[0] < q[2] && q[1] < q[3] && (x0 < 0 || y0 < 0 || x1 > m[2] || y1 > m[1])) return Y5OBB_EINVAL;
      }
    }
    if (ng == 1 && r.n_place[1] != 0) return Y5OBB_EINVAL;
  }
  return Y5OBB_OK;
}

int y5obb_augment_images_u8(const uint8_t* images, const int64_t* meta, int n_images, const y5obb_augment_sample* recs,
                            int B, int S, uint8_t* out, void* stream) {
  if (B <= 0 || S <= 0 || S % 32 || n_images <= 0 || !images || !meta || !recs || !out) return Y5OBB_EINVAL;
  const dim3 blk(32, 8), grd((unsigned)(S / 32), (unsigned)((S + 7) / 8), (unsigned)B);
  k_augment_images<<<grd, blk, 0, (cudaStream_t)stream>>>(images, meta, n_images, recs, S, out);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

size_t y5obb_augment_labels_workspace_bytes(int64_t ncand) { return ncand < 0 ? 0 : labels_ws(ncand, nullptr); }

int y5obb_augment_labels(const float* labels, const int64_t* meta, int n_images, const y5obb_augment_sample* recs,
                         const int64_t* cand_start, int B, int64_t ncand, int S, int nc_theta, double csl_radius, int tcols,
                         float* rows, int64_t* nt, void* workspace, size_t workspace_bytes, void* stream) {
  if (B <= 0 || S <= 0 || S % 32 || n_images <= 0 || ncand < 0 || ncand > INT32_MAX || nc_theta <= 0 ||
      !(csl_radius > 0) || (tcols != 8 && tcols != 7 + nc_theta) || !meta || !recs || !cand_start || !nt)
    return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (ncand == 0) {
    Y5_CUDA(cudaMemsetAsync(nt, 0, sizeof(int64_t), st));
    return Y5OBB_OK;
  }
  if (!labels || !rows || !workspace) return Y5OBB_EINVAL;
  size_t sb = 0;
  if (workspace_bytes < labels_ws(ncand, &sb)) return Y5OBB_EWORKSPACE;
  Carver c(workspace);
  LabelOut* lo = c.take<LabelOut>(ncand);
  int* keep = c.take<int>(ncand);
  int* pos = c.take<int>(ncand);
  void* scan_tmp = c.take<char>(sb);
  const unsigned nb = (unsigned)((ncand + 127) / 128);
  k_augment_labels<<<nb, 128, 0, st>>>(labels, meta, n_images, recs, cand_start, B, ncand, S, lo, keep);
  Y5_LAUNCH_CHECK();
  Y5_CUDA(cub::DeviceScan::InclusiveSum(scan_tmp, sb, keep, pos, (int)ncand, st));
  k_augment_rows<<<nb, 128, 0, st>>>(lo, keep, pos, ncand, nc_theta, csl_radius, tcols, rows, nt);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
