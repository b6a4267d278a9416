// Float polygon NMS and rotated-box overlaps of the DOTA devkit / the nms_rotated extension (SURVEY section 8 rows A14, B4):
//   DOTA_devkit/poly_nms_gpu/poly_nms_kernel.cu:214-264 (K3 kernel), :277-329 (_poly_nms host entry)
//   DOTA_devkit/poly_nms_gpu/poly_overlaps_kernel.cu:283-353 (RotBox2Poly, K4 kernel), :368-427 (_overlaps)
//   utils/nms_rotated/src/poly_nms_cuda.cu:144-261 (K2 = the same kernel behind nms_rotated_ext.nms_poly,
//   unbuildable on torch >= 1.11 because it needs THC)
// All three share one float polygon IoU (triangle fans about the origin, half-plane cuts, eps = 1e-8 sign tests evaluated in
// double).  Parity contract: every floating-point expression below has the operand order and float/double mix of the
// reference expression it restates, and this file is compiled with nvcc's default -fmad=true like the reference, so the
// fused/unfused rounding pattern is the same; tests/test_poly_f32_gpu.py compares IoU matrices bit for bit and keep lists
// against the reference kernels compiled by oracle/build_ref.py for sm_90a (oracle/_ref/libref_polygpu_*.so).
//
// What is NOT the reference's design: only the upper triangle of the 64x64 block grid is evaluated (the reference computes
// the full grid and ignores the lower half), the greedy scan runs on the device (the reference copies the N^2/8-byte matrix
// to the host and scans there), and K2's score sort is a stable CUB radix sort (ties: lower index first).
#include <cub/device/device_radix_sort.cuh>

#include <cstdio>

#include "common.cuh"

// the devkit's host entry points keep the reference's C++ signatures (poly_nms.hpp:9-10, poly_overlaps.hpp:1)
void _poly_nms(int* keep_out, int* num_out, const float* polys_host, int polys_num, int polys_dim, float nms_overlap_thresh,
               int device_id);
void _overlaps(float* overlaps, const float* boxes, const float* query_boxes, int n, int k, int device_id);

namespace y5obb {
namespace {

constexpr int PB = 64;  // polygons per block == bits per mask word
const double kEps = 1E-8;

struct F2 {
  float x, y;
};

// poly_nms_kernel.cu:35-37 (the float argument is compared with a double epsilon)
__device__ __forceinline__ int sgn(float d) { return (d > kEps) - (d < -kEps); }
// :46-48
__device__ __forceinline__ bool same_point(const F2 a, const F2 b) { return sgn(a.x - b.x) == 0 && sgn(a.y - b.y) == 0; }
// :73-75
__device__ __forceinline__ float cross3(F2 o, F2 a, F2 b) { return (a.x - o.x) * (b.y - o.y) - (b.x - o.x) * (a.y - o.y); }
// :76-83 (shoelace over the closed polygon; the division by the double 2.0 is exact)
__device__ __forceinline__ float shoelace(const F2* ps, int n) {
  float res = 0;
  for (int i = 0; i < n; i++) {
    const F2 q = ps[i + 1 == n ? 0 : i + 1];
    res += ps[i].x * q.y - ps[i].y * q.x;
  }
  return res / 2.0;
}
// :84-93; the output point is left untouched when the lines are (numerically) parallel, exactly as the reference leaves it
__device__ __forceinline__ int line_cross(F2 a, F2 b, F2 c, F2 d, F2& p) {
  float s1, s2;
  s1 = cross3(a, b, c);
  s2 = cross3(a, b, d);
  if (sgn(s1) == 0 && sgn(s2) == 0) return 2;
  if (sgn(s2 - s1) == 0) return 0;
  p.x = (c.x * s2 - d.x * s1) / (s2 - s1);
  p.y = (c.y * s2 - d.y * s1) / (s2 - s1);
  return 1;
}

// :118-133: the part of polygon p (n points) to the left of a->b, in place; pp is scratch shared by the three cuts of one
// triangle pair (so a slot line_cross leaves unwritten keeps what the previous cut put there, as in the reference)
__device__ __forceinline__ void cut_left(F2* p, int& n, F2 a, F2 b, F2* pp) {
  int m = 0;
  p[n] = p[0];
  for (int i = 0; i < n; i++) {
    if (sgn(cross3(a, b, p[i])) > 0) pp[m++] = p[i];
    if (sgn(cross3(a, b, p[i])) != sgn(cross3(a, b, p[i + 1]))) line_cross(a, b, p[i], p[i + 1], pp[m++]);
  }
  n = 0;
  for (int i = 0; i < m; i++)
    if (!i || !(same_point(pp[i], pp[i - 1]))) p[n++] = pp[i];
  while (n > 1 && same_point(p[n - 1], p[0])) n--;
}

// :137-154: signed intersection area of the triangles (o, a, b) and (o, c, d), o the origin
__device__ float tri_pair_area(F2 a, F2 b, F2 c, F2 d) {
  F2 o;
  o.x = 0;
  o.y = 0;
  int s1 = sgn(cross3(o, a, b));
  int s2 = sgn(cross3(o, c, d));
  if (s1 == 0 || s2 == 0) return 0.0;
  if (s1 == -1) {
    const F2 t = a;
    a = b;
    b = t;
  }
  if (s2 == -1) {
    const F2 t = c;
    c = d;
    d = t;
  }
  F2 p[10];
  p[0] = o;
  p[1] = a;
  p[2] = b;
#pragma unroll
  for (int i = 3; i < 10; ++i) p[i] = o;  // `float2 p[10] = {o, a, b}` zero-fills the rest
  int n = 3;
  F2 pp[12];
  cut_left(p, n, o, c, pp);
  cut_left(p, n, c, d, pp);
  cut_left(p, n, d, o, pp);
  float res = fabs(shoelace(p, n));
  if (s1 * s2 == -1) res = -res;
  return res;
}

// :156-169: both quadrilaterals made counter-clockwise, then the sum over all edge pairs
__device__ float quad_intersection(F2* ps1, F2* ps2) {
  if (shoelace(ps1, 4) < 0) {
    F2 t = ps1[0];
    ps1[0] = ps1[3];
    ps1[3] = t;
    t = ps1[1];
    ps1[1] = ps1[2];
    ps1[2] = t;
  }
  if (shoelace(ps2, 4) < 0) {
    F2 t = ps2[0];
    ps2[0] = ps2[3];
    ps2[3] = t;
    t = ps2[1];
    ps2[1] = ps2[2];
    ps2[2] = t;
  }
  float res = 0;
  for (int i = 0; i < 4; i++) {
    for (int j = 0; j < 4; j++) {
      res += tri_pair_area(ps1[i], ps1[(i + 1) & 3], ps2[j], ps2[(j + 1) & 3]);
    }
  }
  return res;
}

// :196-217 / poly_overlaps_kernel.cu:306-336: union == 0 -> (inter + 1) / (union + 1)
__device__ __forceinline__ float quad_iou(F2* ps1, F2* ps2) {
  float inter_area = quad_intersection(ps1, ps2);
  float union_area = fabs(shoelace(ps1, 4)) + fabs(shoelace(ps2, 4)) - inter_area;
  float iou = 0;
  if (union_area == 0) {
    iou = (inter_area + 1) / (union_area + 1);
  } else {
    iou = inter_area / union_area;
  }
  return iou;
}

__device__ __forceinline__ float poly_iou(const float* p, const float* q) {
  F2 ps1[4], ps2[4];
  for (int i = 0; i < 4; i++) {
    ps1[i].x = p[i * 2];
    ps1[i].y = p[i * 2 + 1];
    ps2[i].x = q[i * 2];
    ps2[i].y = q[i * 2 + 1];
  }
  return quad_iou(ps1, ps2);
}

// poly_overlaps_kernel.cu:283-303: (cx, cy, w, h, angle) -> corners; float cos/sin, the products in double
__device__ __forceinline__ void rbox_corners(const float* dbox, F2* ps) {
  float cs = cos(dbox[4]);
  float ss = sin(dbox[4]);
  float w = dbox[2];
  float h = dbox[3];
  float x_ctr = dbox[0];
  float y_ctr = dbox[1];
  ps[0].x = x_ctr + cs * (w / 2.0) - ss * (-h / 2.0);
  ps[1].x = x_ctr + cs * (w / 2.0) - ss * (h / 2.0);
  ps[2].x = x_ctr + cs * (-w / 2.0) - ss * (h / 2.0);
  ps[3].x = x_ctr + cs * (-w / 2.0) - ss * (-h / 2.0);
  ps[0].y = y_ctr + ss * (w / 2.0) + cs * (-h / 2.0);
  ps[1].y = y_ctr + ss * (w / 2.0) + cs * (h / 2.0);
  ps[2].y = y_ctr + ss * (-w / 2.0) + cs * (h / 2.0);
  ps[3].y = y_ctr + ss * (-w / 2.0) + cs * (-h / 2.0);
}

// ---- kernels -----------------------------------------------------------------------------------------------------------
// overlaps[x * K + y] = IoU(boxes[x], query[y])  (poly_overlaps_kernel.cu:330-353); y fastest across a warp: coalesced writes
__global__ void k_overlaps(int N, int K, const float* __restrict__ boxes, const float* __restrict__ query, float* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)N * K) return;
  const int x = (int)(t / K), y = (int)(t - (long long)x * K);
  F2 a[4], b[4];
  rbox_corners(boxes + (long long)x * 5, a);
  rbox_corners(query + (long long)y * 5, b);
  out[t] = quad_iou(a, b);
}

__global__ void k_poly_pairs(const float* __restrict__ p8, const float* __restrict__ q8, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = poly_iou(p8 + 8 * i, q8 + 8 * i);
}

__global__ void k_score_keys(const float* __restrict__ dets9, long long n, unsigned int* __restrict__ keys,
                             unsigned int* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned int u = __float_as_uint(dets9[i * 9 + 8] + 0.0f);
  u ^= (u >> 31) ? 0xFFFFFFFFu : 0x80000000u;  // ascending on unsigned compare
  keys[i] = ~u;                                  // descending score
  vals[i] = (unsigned int)i;
}

// Work unit u = (row block rb, column block cb >= rb) of the upper triangle, 64 threads = the rows of rb.
// mask[row * nb + cb] bit c = polygon (cb * 64 + c) of the processing order is suppressed by `row` (IoU > thr), as
// poly_nms_kernel.cu:245-263 writes it.  order == nullptr: the caller's order is the processing order (K3 semantics).
__global__ void __launch_bounds__(PB) k_poly_mask_f32(const float* __restrict__ dets9, const unsigned int* __restrict__ order,
                                                      int n, float thr, unsigned long long* __restrict__ mask) {
  __shared__ float cols[PB * 9];
  const int nb = (n + PB - 1) / PB;
  // u -> (rb, cb): rows are laid out rb = 0 (nb units), rb = 1 (nb - 1 units), ...
  long long u = blockIdx.x;
  int rb = 0;
  while (u >= nb - rb) {
    u -= nb - rb;
    ++rb;
  }
  const int cb = rb + (int)u;
  const int row_size = min(n - rb * PB, PB), col_size = min(n - cb * PB, PB);
  if ((int)threadIdx.x < col_size) {
    const long long src = order ? (long long)order[cb * PB + threadIdx.x] : (long long)(cb * PB + threadIdx.x);
#pragma unroll
    for (int k = 0; k < 9; ++k) cols[threadIdx.x * 9 + k] = dets9[src * 9 + k];
  }
  __syncthreads();
  if ((int)threadIdx.x < row_size) {
    const int row = rb * PB + threadIdx.x;
    const float* cur = dets9 + (order ? (long long)order[row] : (long long)row) * 9;
    unsigned long long t = 0;
    const int start = (rb == cb) ? (int)threadIdx.x + 1 : 0;
    for (int i = start; i < col_size; i++) {
      if (poly_iou(cur, cols + i * 9) > thr) t |= 1ULL << i;
    }
    mask[(long long)row * nb + cb] = t;
  }
}

// Greedy scan of the bit matrix (poly_nms_kernel.cu:306-324) by one CTA: per 64-block the diagonal word chain is resolved
// by one thread, then all threads OR the kept rows' words into the removed set.  keep[k] = order[i] (or i).
__global__ void __launch_bounds__(1024) k_poly_greedy(const unsigned long long* __restrict__ mask,
                                                      const unsigned int* __restrict__ order, int n,
                                                      long long* __restrict__ keep64, int* __restrict__ keep32,
                                                      long long* __restrict__ n_keep64, int* __restrict__ n_keep32) {
  extern __shared__ unsigned long long remv[];
  __shared__ unsigned long long s_diag[PB];
  __shared__ unsigned long long s_kept;
  const int nb = (n + PB - 1) / PB;
  const int tid = threadIdx.x;
  for (int w = tid; w < nb; w += blockDim.x) remv[w] = 0ull;
  __syncthreads();
  long long count = 0;
  for (int blk = 0; blk < nb; ++blk) {
    const int rows = min(PB, n - blk * PB);
    if (tid < PB) s_diag[tid] = tid < rows ? mask[(long long)(blk * PB + tid) * nb + blk] : 0ull;
    __syncthreads();
    if (tid == 0) {
      unsigned long long cur = remv[blk], kept = 0ull;
      if (rows < PB) cur |= ~0ull << rows;
      for (int i = 0; i < PB; ++i) {
        const unsigned long long bit = 1ull << i;
        if (!(cur & bit)) {
          kept |= bit;
          cur |= s_diag[i];
        }
      }
      s_kept = kept;
    }
    __syncthreads();
    const unsigned long long kept = s_kept;
    if (tid < PB && ((kept >> tid) & 1ull)) {
      const long long pos = count + __popcll(kept & ((1ull << tid) - 1ull));
      const int i = blk * PB + tid;
      const long long v = order ? (long long)order[i] : (long long)i;
      if (keep64) keep64[pos] = v;
      if (keep32) keep32[pos] = (int)v;
    }
    count += __popcll(kept);
    for (int w = blk + 1 + tid; w < nb; w += blockDim.x) {
      unsigned long long acc = 0ull, k2 = kept;
      while (k2) {
        const int r = __ffsll((long long)k2) - 1;
        k2 &= k2 - 1;
        acc |= mask[(long long)(blk * PB + r) * nb + w];
      }
      if (acc) remv[w] |= acc;
    }
    __syncthreads();
  }
  if (tid == 0) {
    if (n_keep64) *n_keep64 = count;
    if (n_keep32) *n_keep32 = (int)count;
  }
}

size_t sort_bytes(long long n) {
  size_t b = 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned int*)nullptr, (unsigned int*)nullptr, (const unsigned int*)nullptr,
                                      (unsigned int*)nullptr, (int)n) != cudaSuccess ||
      b == 0) {
    (void)cudaGetLastError();
    b = (size_t)(16u << 20) + (size_t)n * 8;
  }
  return b;
}

int run_poly_nms(const float* dets9, int n, float thr, int presorted, long long* keep64, int* keep32, long long* n64, int* n32,
                 void* ws, size_t ws_bytes, cudaStream_t st) {
  const int nb = (n + PB - 1) / PB;
  if ((size_t)nb * 8 > 200 * 1024) return Y5OBB_EINVAL;  // > 1.6 M polygons
  Carver c(ws);
  unsigned int* keys_a = c.take<unsigned int>(n);
  unsigned int* keys_b = c.take<unsigned int>(n);
  unsigned int* vals_a = c.take<unsigned int>(n);
  unsigned int* vals_b = c.take<unsigned int>(n);
  unsigned long long* mask = c.take<unsigned long long>((size_t)n * nb);
  size_t cub_bytes = sort_bytes(n);
  void* cub_tmp = c.take<char>(cub_bytes);
  if (c.used() > ws_bytes) return Y5OBB_EWORKSPACE;
  const unsigned int* order = nullptr;
  if (!presorted) {
    k_score_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(dets9, n, keys_a, vals_a);
    Y5_LAUNCH_CHECK();
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(cub_tmp, cub_bytes, keys_a, keys_b, vals_a, vals_b, n, 0, 32, st));
    order = vals_b;
  }
  const long long units = (long long)nb * (nb + 1) / 2;
  k_poly_mask_f32<<<(unsigned)units, PB, 0, st>>>(dets9, order, n, thr, mask);
  Y5_LAUNCH_CHECK();
  static bool attr = false;
  if (!attr) {
    Y5_CUDA(cudaFuncSetAttribute(k_poly_greedy, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  k_poly_greedy<<<1, 1024, (size_t)nb * 8, st>>>(mask, order, n, keep64, keep32, n64, n32);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

inline void report(cudaError_t e) {  // the devkit prints CUDA errors to stdout and carries on (poly_nms_kernel.cu:20-27)
  if (e != cudaSuccess) printf("%s\n", cudaGetErrorString(e));
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

size_t y5obb_poly_nms_f32_workspace_bytes(int64_t n) {
  if (n <= 0) return 256;
  const size_t nb = (size_t)((n + PB - 1) / PB);
  return 4096 + (size_t)n * 16 + (size_t)n * nb * 8 + sort_bytes(n);
}

int y5obb_poly_nms_f32(const float* dets9, int64_t n, float iou_thr, int presorted, int64_t* keep_out, int64_t* n_keep_out,
                       void* workspace, size_t workspace_bytes, void* stream) {
  if (n < 0 || !keep_out || !n_keep_out) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    Y5_CUDA(cudaMemsetAsync(n_keep_out, 0, sizeof(int64_t), st));
    return Y5OBB_OK;
  }
  if (!dets9 || !workspace || n > 1000000) return Y5OBB_EINVAL;
  return run_poly_nms(dets9, (int)n, iou_thr, presorted, reinterpret_cast<long long*>(keep_out), nullptr,
                      reinterpret_cast<long long*>(n_keep_out), nullptr, workspace, workspace_bytes, st);
}

int y5obb_poly_overlaps_f32(const float* boxes5, const float* query5, int64_t n, int64_t k, float* overlaps, void* stream) {
  if (n < 0 || k < 0) return Y5OBB_EINVAL;
  if (n == 0 || k == 0) return Y5OBB_OK;
  if (!boxes5 || !query5 || !overlaps || n > 0x7FFFFFFF || k > 0x7FFFFFFF) return Y5OBB_EINVAL;
  const long long total = (long long)n * k;
  k_overlaps<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>((int)n, (int)k, boxes5, query5, overlaps);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_poly_iou_pairs_f32(const float* p8, const float* q8, float* iou_out, int64_t n, void* stream) {
  if (n < 0) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  if (!p8 || !q8 || !iou_out) return Y5OBB_EINVAL;
  k_poly_pairs<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(p8, q8, iou_out, n);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"

// ---- the devkit's own entry points (host pointers, synchronous, default stream; C++ linkage as in the reference headers) ----
void _poly_nms(int* keep_out, int* num_out, const float* polys_host, int polys_num, int polys_dim, float nms_overlap_thresh,
               int device_id) {
  if (num_out) *num_out = 0;
  if (polys_num <= 0 || !keep_out || !num_out || !polys_host) return;
  if (polys_dim != 9) {  // the reference kernel hard-codes 9 floats per polygon (poly_nms_kernel.cu:229-247)
    printf("_poly_nms: polys_dim must be 9\n");
    return;
  }
  int cur = 0;
  report(cudaGetDevice(&cur));
  if (cur != device_id) report(cudaSetDevice(device_id));
  float* polys_dev = nullptr;
  char* ws = nullptr;
  int* keep_dev = nullptr;
  const size_t ws_bytes = y5obb_poly_nms_f32_workspace_bytes(polys_num);
  report(cudaMalloc(&polys_dev, (size_t)polys_num * 9 * sizeof(float)));
  report(cudaMalloc(&ws, ws_bytes));
  report(cudaMalloc(&keep_dev, ((size_t)polys_num + 1) * sizeof(int)));
  if (polys_dev && ws && keep_dev) {
    report(cudaMemcpy(polys_dev, polys_host, (size_t)polys_num * 9 * sizeof(float), cudaMemcpyHostToDevice));
    // the caller's order IS the processing order (poly_nms.pyx sorts by score before calling)
    const int rc = run_poly_nms(polys_dev, polys_num, nms_overlap_thresh, 1, nullptr, keep_dev + 1, nullptr, keep_dev, ws, ws_bytes,
                                (cudaStream_t)0);
    if (rc != Y5OBB_OK) printf("_poly_nms: kernel launch failed (%d)\n", rc);
    int cnt = 0;
    report(cudaMemcpy(&cnt, keep_dev, sizeof(int), cudaMemcpyDeviceToHost));
    if (rc == Y5OBB_OK && cnt > 0 && cnt <= polys_num) {
      report(cudaMemcpy(keep_out, keep_dev + 1, (size_t)cnt * sizeof(int), cudaMemcpyDeviceToHost));
      *num_out = cnt;
    }
  }
  if (polys_dev) report(cudaFree(polys_dev));
  if (ws) report(cudaFree(ws));
  if (keep_dev) report(cudaFree(keep_dev));
}

void _overlaps(float* overlaps, const float* boxes, const float* query_boxes, int n, int k, int device_id) {
  if (n <= 0 || k <= 0 || !overlaps || !boxes || !query_boxes) return;
  int cur = 0;
  report(cudaGetDevice(&cur));
  if (cur != device_id) report(cudaSetDevice(device_id));
  float *ov = nullptr, *b = nullptr, *q = nullptr;
  report(cudaMalloc(&b, (size_t)n * 5 * sizeof(float)));
  report(cudaMalloc(&q, (size_t)k * 5 * sizeof(float)));
  report(cudaMalloc(&ov, (size_t)n * k * sizeof(float)));
  if (b && q && ov) {
    report(cudaMemcpy(b, boxes, (size_t)n * 5 * sizeof(float), cudaMemcpyHostToDevice));
    report(cudaMemcpy(q, query_boxes, (size_t)k * 5 * sizeof(float), cudaMemcpyHostToDevice));
    const int rc = y5obb_poly_overlaps_f32(b, q, n, k, ov, nullptr);
    if (rc != Y5OBB_OK) printf("_overlaps: kernel launch failed (%d)\n", rc);
    report(cudaMemcpy(overlaps, ov, (size_t)n * k * sizeof(float), cudaMemcpyDeviceToHost));
  }
  if (ov) report(cudaFree(ov));
  if (b) report(cudaFree(b));
  if (q) report(cudaFree(q));
}

extern "C" {
// C-linkage aliases of the two devkit entry points for ctypes / cgo style bindings
void y5obb_devkit_poly_nms(int* keep_out, int* num_out, const float* polys_host, int polys_num, int polys_dim, float thresh,
                           int device_id) {
  _poly_nms(keep_out, num_out, polys_host, polys_num, polys_dim, thresh, device_id);
}
void y5obb_devkit_overlaps(float* overlaps, const float* boxes, const float* query_boxes, int n, int k, int device_id) {
  _overlaps(overlaps, boxes, query_boxes, n, k, device_id);
}
}
