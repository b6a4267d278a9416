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
#include "geom.cuh"

namespace y5obb {
namespace {

using namespace geom;

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
  const unsigned long long bits =
      poly_suppress_word([&](long long j) { return dets9 + (long long)order[j] * 9; }, i, w, n, thresh);
  mask[i * words + w] = bits;
}

__global__ void k_poly_reduce(const unsigned long long* __restrict__ mask, const unsigned int* __restrict__ order, long long n,
                              long long* __restrict__ keep, long long* __restrict__ n_keep) {
  extern __shared__ unsigned long long remv[];
  const long long k = poly_greedy_scan(mask, n, remv, [&](long long slot, long long i) { keep[slot] = (long long)order[i]; });
  if (threadIdx.x == 0) *n_keep = k;
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
