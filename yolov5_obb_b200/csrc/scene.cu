// Whole-scene DOTA inference around the per-tile engine (README.md:24-26 / docs/GetStart.md:117-130 of the reference):
//   y5obb_scene_tiles_s2d_u8  DOTA_devkit/ImgSplit_multi_process.py:122-132,226-273 (crop, zero padding beyond the scene)
//                             + utils/augmentations.py:92-128 letterbox (114 border, auto=False, scaleup=False)
//                             + utils/datasets.py BGR -> RGB + the `/ 255` and 2x2 space-to-depth layout of k_stem_s2d_u8:
//                             the stem input of every tile, straight from the decoded scene (no tile is ever materialised).
//   y5obb_scene_merge_f64     val.py:50-66 save_one_json (rbox2poly, scale_polys, round(x, 1), round(conf, 5)),
//                             DOTA_devkit/ResultMerge_multi_process.py:175-182 poly2origpoly and :62-123,158-174
//                             py_cpu_nms_poly_fast per class, all classes of the scene in one pass.
//
// Merge pipeline: k_merge_keys (one 64-bit key per detection: class | 100000 - round(conf * 1e5) | tile * max_det + row, so
// that one radix sort yields the class segments in descending rounded score, ties -> lower (tile, row)) -> CUB radix sort ->
// k_merge_build (scene-space fp64 polygons in sorted order) -> the per-class candidate counts are read by the host (the one
// synchronisation: they size the dense suppression masks) -> k_merge_mask (every class segment in one launch) ->
// k_merge_reduce (one block per class: greedy scan) -> k_merge_gather ([K, 10] rows, per class in keep order).
#include <cuda_bf16.h>

#include <algorithm>
#include <cub/cub.cuh>

#include "common.cuh"
#include "geom.cuh"
#include "stage.cuh"

namespace y5obb {
namespace {

using namespace geom;

template <typename E>
__global__ void k_scene_tiles_s2d_u8(const uint8_t* __restrict__ scene, long long H, long long W,
                                     const int32_t* __restrict__ origins, int T, int S, int size, int border,
                                     E* __restrict__ out, int pad_cols) {
  const int Ho = size >> 1, Wo = size >> 1;
  const long long total = (long long)T * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long r = i / Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    const long long left = origins[2 * b], up = origins[2 * b + 1];
    float v[16];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int y = 2 * ho + (d >> 1) - border, x = 2 * wo + (d & 1) - border;  // tile pixel under the letterbox border
      uint8_t px[3] = {114, 114, 114};
      if (y >= 0 && y < S && x >= 0 && x < S) {
        const long long sy = up + y, sx = left + x;
        if (sy >= 0 && sy < H && sx >= 0 && sx < W) {
          const uint8_t* p = scene + (sy * W + sx) * 3;
          px[0] = p[2];  // BGR -> RGB
          px[1] = p[1];
          px[2] = p[0];
        } else {
          px[0] = px[1] = px[2] = 0;  // ImgSplit's zero padding of tiles that reach beyond the scene
        }
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) v[d * 3 + c] = u8_value(px[c], out);
    }
    v[12] = v[13] = v[14] = v[15] = 0.f;
    uint4 o[2];
    pack16(v, out, o);
    uint4* dst = reinterpret_cast<uint4*>(out + ((r * (Wo + 2 * pad_cols)) + wo + pad_cols) * 16);
    dst[0] = o[0];
    dst[1] = o[1];
  }
}

constexpr int KEY_CLS_SHIFT = 57, KEY_SCORE_SHIFT = 40;
constexpr unsigned long long KEY_SLOT_MASK = (1ull << KEY_SCORE_SHIFT) - 1;
constexpr unsigned long long KEY_NONE = ~0ull;

__global__ void k_merge_keys(const float* __restrict__ rows7, const int64_t* __restrict__ counts, long long n_slots, int max_det,
                             int nc, unsigned long long* __restrict__ keys, long long* __restrict__ cls_cnt) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const long long t = s / max_det, r = s - t * max_det;
  unsigned long long key = KEY_NONE;
  if (r < counts[t]) {
    const float* row = rows7 + s * 7;
    const int cls = (int)row[6];
    const double k = py_round_int((double)row[5], 1e5);  // round(conf, 5) * 1e5: orders the rounded scores exactly
    if (cls >= 0 && cls < nc && k >= 0.0 && k <= 100000.0) {
      key = ((unsigned long long)cls << KEY_CLS_SHIFT) | ((unsigned long long)(100000.0 - k) << KEY_SCORE_SHIFT) |
            (unsigned long long)s;
      atomicAdd(reinterpret_cast<unsigned long long*>(cls_cnt + cls), 1ull);
    }
  }
  keys[s] = key;
}

// sorted position p -> dets9[p] = scene-space polygon (8 fp64) + rounded score, as the reference's merge reads them back
__global__ void k_merge_build(const float* __restrict__ rows7, const int32_t* __restrict__ origins, const unsigned long long* __restrict__ keys,
                              long long n_slots, int max_det, float pad, float gain, double* __restrict__ dets9) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_slots) return;
  const unsigned long long key = keys[p];
  if (key == KEY_NONE) return;
  const long long s = (long long)(key & KEY_SLOT_MASK), t = s / max_det;
  const float* row = rows7 + s * 7;
  float poly[8];
  rbox2poly_f32(row[0], row[1], row[2], row[3], row[4], poly);
  const double org[2] = {(double)origins[2 * t], (double)origins[2 * t + 1]};
  double* d = dets9 + p * 9;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float v = __fdiv_rn(__fsub_rn(poly[k], pad), gain);       // scale_polys (general.py:636-650)
    d[k] = __dadd_rn(py_round((double)v, 10.0), org[k & 1]);          // round(x, 1) (val.py:65), then (x + left) / 1.0
  }
  d[8] = py_round((double)row[5], 1e5);                                // round(conf, 5) (val.py:64)
}

constexpr int MAX_NC = 64;
struct SegTable {
  long long start[MAX_NC + 1];     // first sorted position of class c (start[nc] = candidates)
  long long mask_off[MAX_NC + 1];  // first mask word of class c
};

__device__ __forceinline__ int seg_of(const long long* off, int nc, long long x) {  // largest c with off[c] <= x
  int lo = 0, hi = nc - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void k_merge_mask(const double* __restrict__ dets9, const __grid_constant__ SegTable tab, int nc, double thresh,
                             unsigned long long* __restrict__ mask) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= tab.mask_off[nc]) return;
  const int c = seg_of(tab.mask_off, nc, t);
  const long long n = tab.start[c + 1] - tab.start[c], words = (n + 63) / 64;
  const long long local = t - tab.mask_off[c], i = local / words, w = local - i * words;
  const double* base = dets9 + tab.start[c] * 9;
  mask[t] = poly_suppress_word([&](long long j) { return base + j * 9; }, i, w, n, thresh);
}

__global__ void k_merge_reduce(const unsigned long long* __restrict__ mask, const __grid_constant__ SegTable tab,
                               long long* __restrict__ keep_pos, long long* __restrict__ keep_cnt) {
  extern __shared__ unsigned long long remv[];
  const int c = blockIdx.x;
  const long long s0 = tab.start[c], n = tab.start[c + 1] - s0;
  const long long k = poly_greedy_scan(mask + tab.mask_off[c], n, remv, [&](long long slot, long long i) { keep_pos[s0 + slot] = s0 + i; });
  if (threadIdx.x == 0) keep_cnt[c] = k;
}

__global__ void k_merge_gather(const double* __restrict__ dets9, const __grid_constant__ SegTable tab, int nc,
                               const long long* __restrict__ keep_pos, const long long* __restrict__ keep_cnt,
                               double* __restrict__ out10, int64_t* __restrict__ n_out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p == 0) {
    long long k = 0;
    for (int c = 0; c < nc; ++c) k += keep_cnt[c];
    *n_out = k;
  }
  if (p >= tab.start[nc]) return;
  const int c = seg_of(tab.start, nc, p);
  const long long j = p - tab.start[c];
  if (j >= keep_cnt[c]) return;
  long long o = j;
  for (int q = 0; q < c; ++q) o += keep_cnt[q];
  const double* d = dets9 + keep_pos[p] * 9;
  double* r = out10 + o * 10;
  r[0] = (double)c;
  r[1] = d[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[2 + k] = d[k];
}

size_t sort_bytes(long long n) {
  size_t b = 0;
  if (cub::DeviceRadixSort::SortKeys(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n) !=
      cudaSuccess) {
    (void)cudaGetLastError();
    b = (size_t)(32u << 20) + (size_t)n * 16;
  }
  return b;
}

// workspace carve of the merge; the class masks come last (their size is known only after the candidate counts are read)
struct MergeWs {
  unsigned long long *keys_in, *keys_out;
  long long *cls_cnt, *keep_pos, *keep_cnt;
  double* dets9;
  void* sort_tmp;
  size_t sort_tmp_bytes;
  unsigned long long* mask;
  size_t fixed;
  MergeWs(void* base, long long n_slots, int nc) {
    Carver c(base);
    keys_in = c.take<unsigned long long>(n_slots);
    keys_out = c.take<unsigned long long>(n_slots);
    cls_cnt = c.take<long long>(nc);
    keep_cnt = c.take<long long>(nc);
    keep_pos = c.take<long long>(n_slots);
    dets9 = c.take<double>((size_t)n_slots * 9);
    sort_tmp_bytes = sort_bytes(n_slots);
    sort_tmp = c.take<char>(sort_tmp_bytes);
    fixed = c.used();
    mask = reinterpret_cast<unsigned long long*>(static_cast<char*>(base) + fixed);
  }
};

size_t mask_words(const int64_t* class_cands_host, int nc) {
  size_t w = 0;
  for (int c = 0; c < nc; ++c) w += (size_t)class_cands_host[c] * (size_t)((class_cands_host[c] + 63) / 64);
  return w;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

static int scene_tiles_s2d_u8(bool f16, const uint8_t* scene_hwc, int64_t H, int64_t W, const int32_t* origins2, int n_tiles,
                              int subsize, int size, int border, void* out_nhwc16, int pad_cols, void* stream) {
  if (!scene_hwc || !origins2 || !out_nhwc16 || H <= 0 || W <= 0 || n_tiles <= 0 || subsize <= 0 || (size & 1) || size <= 0 ||
      border < 0 || border + subsize > size || pad_cols < 0)
    return Y5OBB_EINVAL;
  if (reinterpret_cast<uintptr_t>(out_nhwc16) & 15) return Y5OBB_EINVAL;
  const long long total = (long long)n_tiles * (size / 2) * (size / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  if (f16)
    k_scene_tiles_s2d_u8<<<grid, 256, 0, (cudaStream_t)stream>>>(scene_hwc, H, W, origins2, n_tiles, subsize, size, border,
                                                                static_cast<__half*>(out_nhwc16), pad_cols);
  else
    k_scene_tiles_s2d_u8<<<grid, 256, 0, (cudaStream_t)stream>>>(scene_hwc, H, W, origins2, n_tiles, subsize, size, border,
                                                                static_cast<__nv_bfloat16*>(out_nhwc16), pad_cols);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_scene_tiles_s2d_u8(const uint8_t* scene_hwc, int64_t H, int64_t W, const int32_t* origins2, int n_tiles, int subsize,
                             int size, int border, void* out_nhwc16, int pad_cols, void* stream) {
  return scene_tiles_s2d_u8(false, scene_hwc, H, W, origins2, n_tiles, subsize, size, border, out_nhwc16, pad_cols, stream);
}

int y5obb_scene_tiles_s2d_u8_f16(const uint8_t* scene_hwc, int64_t H, int64_t W, const int32_t* origins2, int n_tiles,
                                 int subsize, int size, int border, void* out_nhwc16, int pad_cols, void* stream) {
  return scene_tiles_s2d_u8(true, scene_hwc, H, W, origins2, n_tiles, subsize, size, border, out_nhwc16, pad_cols, stream);
}

size_t y5obb_scene_merge_workspace_bytes(int64_t n_tiles, int max_det, int nc, const int64_t* class_cands_host) {
  if (n_tiles <= 0 || max_det <= 0 || nc <= 0 || nc > MAX_NC) return 256;
  const long long n_slots = n_tiles * (long long)max_det;
  char probe;  // (only the offsets are used)
  MergeWs ws(&probe, n_slots, nc);
  return ws.fixed + (class_cands_host ? mask_words(class_cands_host, nc) * 8 : 0) + 256;
}

int y5obb_scene_merge_f64(const float* rows7, const int64_t* counts, const int32_t* origins2, int64_t n_tiles, int max_det,
                          int nc, float pad, float gain, double thresh, double* out10, int64_t* n_out,
                          int64_t* class_cands_host, void* workspace, size_t workspace_bytes, void* stream) {
  if (!rows7 || !counts || !origins2 || !out10 || !n_out || !class_cands_host || !workspace || n_tiles <= 0 || max_det <= 0 ||
      nc <= 0 || nc > MAX_NC || !(gain > 0.0f))
    return Y5OBB_EINVAL;
  const long long n_slots = n_tiles * (long long)max_det;
  if (n_slots > (long long)KEY_SLOT_MASK || n_slots > 0x7FFFFFFFll) return Y5OBB_EINVAL;
  if (y5obb_scene_merge_workspace_bytes(n_tiles, max_det, nc, nullptr) > workspace_bytes) return Y5OBB_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  MergeWs ws(workspace, n_slots, nc);
  const unsigned g = (unsigned)((n_slots + 255) / 256);
  Y5_CUDA(cudaMemsetAsync(ws.cls_cnt, 0, sizeof(long long) * nc, st));
  k_merge_keys<<<g, 256, 0, st>>>(rows7, counts, n_slots, max_det, nc, ws.keys_in, ws.cls_cnt);
  Y5_LAUNCH_CHECK();
  size_t tmp = ws.sort_tmp_bytes;
  Y5_CUDA(cub::DeviceRadixSort::SortKeys(ws.sort_tmp, tmp, ws.keys_in, ws.keys_out, (int)n_slots, 0, 64, st));
  k_merge_build<<<g, 256, 0, st>>>(rows7, origins2, ws.keys_out, n_slots, max_det, pad, gain, ws.dets9);
  Y5_LAUNCH_CHECK();
  // the one host read: per-class candidate counts size the dense masks
  Y5_CUDA(cudaMemcpyAsync(class_cands_host, ws.cls_cnt, sizeof(int64_t) * nc, cudaMemcpyDeviceToHost, st));
  Y5_CUDA(cudaStreamSynchronize(st));
  SegTable tab{};
  for (int c = 0; c < nc; ++c) {
    if (class_cands_host[c] > Y5OBB_SCENE_MAX_CLASS_CANDIDATES) return Y5OBB_EINVAL;
    tab.start[c + 1] = tab.start[c] + class_cands_host[c];
    tab.mask_off[c + 1] = tab.mask_off[c] + class_cands_host[c] * ((class_cands_host[c] + 63) / 64);
  }
  if (y5obb_scene_merge_workspace_bytes(n_tiles, max_det, nc, class_cands_host) > workspace_bytes) return Y5OBB_EWORKSPACE;
  if (tab.start[nc] == 0) {
    Y5_CUDA(cudaMemsetAsync(n_out, 0, sizeof(int64_t), st));
    return Y5OBB_OK;
  }
  long long max_n = 0;
  for (int c = 0; c < nc; ++c) max_n = std::max<long long>(max_n, class_cands_host[c]);
  k_merge_mask<<<(unsigned)((tab.mask_off[nc] + 127) / 128), 128, 0, st>>>(ws.dets9, tab, nc, thresh, ws.mask);
  Y5_LAUNCH_CHECK();
  k_merge_reduce<<<nc, 1024, (size_t)((max_n + 63) / 64) * 8, st>>>(ws.mask, tab, ws.keep_pos, ws.keep_cnt);
  Y5_LAUNCH_CHECK();
  k_merge_gather<<<(unsigned)((tab.start[nc] + 255) / 256), 256, 0, st>>>(ws.dets9, tab, nc, ws.keep_pos, ws.keep_cnt, out10,
                                                                          n_out);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
