// DOTA Task1 evaluation (DOTA_devkit/dota_evaluation_task1.py:54-249, voc_ap and voc_eval) for every class in one call:
//   y5obb_dota_eval_f64    the per-class matching, precision / recall curve and VOC AP, bit for bit, without a host read.
//   y5obb_task1_round_f64  write_task1's round(score, 2) / round(x, 1) on merged scene rows (the in-memory route).
//
// Pipeline: k_eval_det_keys (descending-score keys, class buckets, class counts) -> CUB radix sort by score, then a stable
// sort by class (ties -> lower input index) -> k_eval_offsets (class_off) ; k_eval_gt_keys ((class, image) keys, npos) -> CUB
// radix sort (file order within a key) -> k_eval_match (one thread per sorted detection: its (image, class) GT segment, the
// axis-aligned pre-filter, iou_poly_dev, ovmax / jmax, the first matching position per GT by atomicMin) -> k_eval_tpfp ->
// CUB inclusive scan of packed (tp, fp) counts -> k_eval_curve (rec, prec) -> k_eval_ap (one block per class).
//
// TP / FP without voc_eval's sequential loop: R['det'] changes only on a true positive, so a detection is TP exactly when
// ovmax > ovthresh, GT jmax is not difficult and no earlier detection (in sorted order) has that same GT as its match; later
// matches to a non-difficult GT are FP, matches to a difficult GT are neither.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cub/cub.cuh>

#include "common.cuh"
#include "geom.cuh"
#include "np_sum.cuh"

namespace y5obb {
namespace {

using namespace geom;

constexpr long long MATCH_FP = -1, MATCH_IGNORED = -2;

// ascending order of the key = descending score; NaN last (argsort of -confidence puts NaN last), -0.0 ties with +0.0
__device__ __forceinline__ unsigned long long desc_score_key(double s) {
  if (isnan(s)) return ~0ull;
  const unsigned long long b = (unsigned long long)__double_as_longlong(__dadd_rn(s, 0.0));
  const unsigned long long asc = (b >> 63) ? ~b : (b | (1ull << 63));
  return ~asc;
}

// numpy's minimum / maximum (and min / max reductions): NaN propagates
__device__ __forceinline__ double np_min(double a, double b) { return (a < b || isnan(a)) ? a : b; }
__device__ __forceinline__ double np_max(double a, double b) { return (a > b || isnan(a)) ? a : b; }

__device__ __forceinline__ int det_class(const double* det10, long long i, int nc, int n_images, const int32_t* det_img) {
  const double c = det10[i * 10];
  const int img = det_img[i];
  if (!(c >= 0.0 && c < (double)nc && c == floor(c)) || img < 0 || img >= n_images) return -1;
  return (int)c;
}

__global__ void k_eval_det_keys(const int32_t* __restrict__ det_img, const double* __restrict__ det10, long long n, int nc,
                                int n_images, unsigned long long* __restrict__ score_key, int* __restrict__ idx,
                                long long* __restrict__ cls_cnt, int32_t* __restrict__ status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  score_key[i] = desc_score_key(det10[i * 10 + 1]);
  idx[i] = (int)i;
  const int c = det_class(det10, i, nc, n_images, det_img);
  if (c < 0) *status = Y5OBB_EINVAL;
  else atomicAdd(reinterpret_cast<unsigned long long*>(cls_cnt + c), 1ull);
}

// class bucket of the score-sorted detections (nc for an invalid row: they sort past every class segment)
__global__ void k_eval_cls_keys(const int32_t* __restrict__ det_img, const double* __restrict__ det10, long long n, int nc,
                                int n_images, const int* __restrict__ idx, unsigned* __restrict__ cls_key) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int c = det_class(det10, idx[p], nc, n_images, det_img);
  cls_key[p] = c < 0 ? (unsigned)nc : (unsigned)c;
}

__global__ void k_eval_offsets(const long long* __restrict__ cls_cnt, int nc, int64_t* __restrict__ class_off) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  long long s = 0;
  class_off[0] = 0;
  for (int c = 0; c < nc; ++c) class_off[c + 1] = (s += cls_cnt[c]);
}

__global__ void k_eval_gt_keys(const int32_t* __restrict__ gt_img, const double* __restrict__ gt10, long long n, int nc,
                               int n_images, unsigned long long* __restrict__ key, int* __restrict__ idx,
                               int64_t* __restrict__ npos, int* __restrict__ first_pos, int32_t* __restrict__ status) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double c = gt10[j * 10];
  const int img = gt_img[j];
  idx[j] = (int)j;
  first_pos[j] = INT_MAX;
  if (!(c >= 0.0 && c < (double)nc && c == floor(c)) || img < 0 || img >= n_images) {
    *status = Y5OBB_EINVAL;
    key[j] = (unsigned long long)nc * (unsigned long long)n_images;  // past every (class, image) key
    return;
  }
  key[j] = (unsigned long long)c * (unsigned long long)n_images + (unsigned long long)img;
  if (gt10[j * 10 + 1] == 0.0) atomicAdd(reinterpret_cast<unsigned long long*>(npos + (int)c), 1ull);  // sum(~difficult)
}

__device__ __forceinline__ long long lower_bound(const unsigned long long* a, long long n, unsigned long long k) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct Box {
  double x0, y0, x1, y1;  // np.min / np.max of the x and y coordinates
};
__device__ __forceinline__ Box hbb(const double* p8) {
  Box b{p8[0], p8[1], p8[0], p8[1]};
  for (int k = 1; k < 4; ++k) {
    b.x0 = np_min(b.x0, p8[2 * k]);
    b.x1 = np_max(b.x1, p8[2 * k]);
    b.y0 = np_min(b.y0, p8[2 * k + 1]);
    b.y1 = np_max(b.y1, p8[2 * k + 1]);
  }
  return b;
}

// dota_evaluation_task1.py:167-231 for sorted position p: match[p] = the GT it claims (global index), MATCH_FP or MATCH_IGNORED
__global__ void k_eval_match(const int32_t* __restrict__ det_img, const double* __restrict__ det10, long long n_det,
                             const double* __restrict__ gt10, const unsigned long long* __restrict__ gt_key,
                             const int* __restrict__ gt_idx, long long n_gt, int n_images, const int* __restrict__ perm,
                             const int64_t* __restrict__ class_off, int nc, double ovthresh, long long* __restrict__ match,
                             int* __restrict__ first_pos) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_det || p >= class_off[nc]) return;
  const int d = perm[p];
  const unsigned long long key = (unsigned long long)det10[(long long)d * 10] * (unsigned long long)n_images +
                                 (unsigned long long)det_img[d];
  const long long lo = lower_bound(gt_key, n_gt, key), hi = lower_bound(gt_key, n_gt, key + 1);
  const double* bb = det10 + (long long)d * 10 + 2;
  const Box b = hbb(bb);
  const double barea = __dmul_rn(__dadd_rn(__dsub_rn(b.x1, b.x0), 1.0), __dadd_rn(__dsub_rn(b.y1, b.y0), 1.0));
  double ovmax = -INFINITY;
  long long jmax = -1;
  for (long long q = lo; q < hi; ++q) {
    const int j = gt_idx[q];
    const double* g8 = gt10 + (long long)j * 10 + 2;
    const Box g = hbb(g8);
    // :189-206, the +1 pixel convention on the intersection and on both areas of the union
    const double iw = np_max(__dadd_rn(__dsub_rn(np_min(g.x1, b.x1), np_max(g.x0, b.x0)), 1.0), 0.0);
    const double ih = np_max(__dadd_rn(__dsub_rn(np_min(g.y1, b.y1), np_max(g.y0, b.y0)), 1.0), 0.0);
    const double inters = __dmul_rn(iw, ih);
    const double garea = __dmul_rn(__dadd_rn(__dsub_rn(g.x1, g.x0), 1.0), __dadd_rn(__dsub_rn(g.y1, g.y0), 1.0));
    const double uni = __dsub_rn(__dadd_rn(barea, garea), inters);
    if (!(__ddiv_rn(inters, uni) > 0.0)) continue;
    const double ov = iou_poly_dev(g8, bb);  // :212 iou_poly(GT, det), in that order
    // np.max / np.argmax over the kept GTs in file order: the first NaN wins and sticks, else the first maximum
    if (jmax < 0 || (!isnan(ovmax) && (isnan(ov) || ov > ovmax))) {
      ovmax = ov;
      jmax = j;
    }
  }
  long long m = MATCH_FP;
  if (ovmax > ovthresh) {
    if (gt10[jmax * 10 + 1] != 0.0) {
      m = MATCH_IGNORED;
    } else {
      m = jmax;
      atomicMin(first_pos + jmax, (int)p);
    }
  }
  match[p] = m;
}

// packed (tp << 32 | fp) per sorted position; 0 past the valid rows
__global__ void k_eval_tpfp(const long long* __restrict__ match, const int* __restrict__ first_pos, long long n_det,
                            const int64_t* __restrict__ class_off, int nc, unsigned long long* __restrict__ tpfp) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_det) return;
  unsigned long long v = 0;
  if (p < class_off[nc]) {
    const long long m = match[p];
    if (m == MATCH_FP) v = 1;
    else if (m >= 0) v = first_pos[m] == (int)p ? (1ull << 32) : 1ull;
  }
  tpfp[p] = v;
}

__device__ __forceinline__ int class_of(const int64_t* off, int nc, long long p) {  // largest c with off[c] <= p
  int lo = 0, hi = nc - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// :240-246: cumulative tp / fp within the class (exact integers), rec = tp / npos, prec = tp / max(tp + fp, eps)
__global__ void k_eval_curve(const unsigned long long* __restrict__ csum, long long n_det, const int64_t* __restrict__ class_off,
                             int nc, const int64_t* __restrict__ npos, double* __restrict__ rec, double* __restrict__ prec) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_det || p >= class_off[nc]) return;
  const int c = class_of(class_off, nc, p);
  const long long s = class_off[c];
  const unsigned long long v = csum[p] - (s > 0 ? csum[s - 1] : 0ull);
  const double tp = (double)(v >> 32), fp = (double)(v & 0xffffffffull);
  rec[p] = __ddiv_rn(tp, (double)npos[c]);
  prec[p] = __ddiv_rn(tp, fmax(__dadd_rn(tp, fp), DBL_EPSILON));
}

constexpr int AP_THREADS = 256;

// voc_ap (:54-85), one block per class; scratch holds n + 2 doubles of this class
__global__ void __launch_bounds__(AP_THREADS) k_eval_ap(const double* __restrict__ rec_all, const double* __restrict__ prec_all,
                                                        const int64_t* __restrict__ class_off, int use_07_metric,
                                                        double* __restrict__ scratch_all, double* __restrict__ ap) {
  const int c = blockIdx.x;
  const long long s = class_off[c], n = class_off[c + 1] - s;
  const double* rec = rec_all + s;
  const double* prec = prec_all + s;
  if (use_07_metric) {
    // p_k = max(prec[rec >= k * 0.1]) or 0; prec >= 0, so -1 marks an empty selection
    __shared__ double red[11][AP_THREADS];
    double pm[11];
    for (int k = 0; k < 11; ++k) pm[k] = -1.0;
    for (long long i = threadIdx.x; i < n; i += AP_THREADS)
      for (int k = 0; k < 11; ++k)
        if (rec[i] >= __dmul_rn((double)k, 0.1)) pm[k] = fmax(pm[k], prec[i]);
    for (int k = 0; k < 11; ++k) red[k][threadIdx.x] = pm[k];
    __syncthreads();
    for (int w = AP_THREADS / 2; w > 0; w >>= 1) {
      if (threadIdx.x < w)
        for (int k = 0; k < 11; ++k) red[k][threadIdx.x] = fmax(red[k][threadIdx.x], red[k][threadIdx.x + w]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      double a = 0.0;
      for (int k = 0; k < 11; ++k) a = __dadd_rn(a, __ddiv_rn(red[k][0] < 0.0 ? 0.0 : red[k][0], 11.0));
      ap[c] = a;
    }
    return;
  }
  if (threadIdx.x != 0) return;
  // mpre = [0, prec, 0] with its suffix-max envelope; mrec = [0, rec, 1]
  double* env = scratch_all + s + 2ll * c;
  env[n + 1] = 0.0;
  for (long long i = n; i >= 1; --i) env[i] = np_max(prec[i - 1], env[i + 1]);
  env[0] = np_max(0.0, env[1]);
  // terms (mrec[i + 1] - mrec[i]) * mpre[i + 1] where mrec changes (NaN compares unequal), compacted in place: the write
  // index never passes the next read index
  long long m = 0;
  for (long long i = 0; i <= n; ++i) {
    const double r0 = i == 0 ? 0.0 : rec[i - 1];
    const double r1 = i == n ? 1.0 : rec[i];
    if (r1 != r0) env[m++] = __dmul_rn(__dsub_rn(r1, r0), env[i + 1]);
  }
  ap[c] = np_pairwise_sum(env, m);
}

__global__ void k_task1_round(const double* __restrict__ in10, long long n, double* __restrict__ out10) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* r = in10 + i * 10;
  double* o = out10 + i * 10;
  o[0] = r[0];
  o[1] = py_round(r[1], 100.0);                            // str(round(score, 2))
  for (int k = 2; k < 10; ++k) o[k] = py_round(r[k], 10.0);  // str(round(x, 1))
}

int bit_length(unsigned long long v) {
  int b = 0;
  while (v) {
    ++b;
    v >>= 1;
  }
  return b < 1 ? 1 : b;
}

template <typename K>
size_t sort_pairs_bytes(long long n) {
  size_t b = 0;
  if (n <= 0) return 0;
  if (cub::DeviceRadixSort::SortPairs(nullptr, b, (const K*)nullptr, (K*)nullptr, (const int*)nullptr, (int*)nullptr, (int)n) !=
      cudaSuccess) {
    (void)cudaGetLastError();
    b = (size_t)(32u << 20) + (size_t)n * 16;
  }
  return b;
}

size_t scan_bytes(long long n) {
  size_t b = 0;
  if (n <= 0) return 0;
  if (cub::DeviceScan::InclusiveSum(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n) !=
      cudaSuccess) {
    (void)cudaGetLastError();
    b = (size_t)(32u << 20) + (size_t)n * 16;
  }
  return b;
}

struct EvalWs {
  unsigned long long *dkey_in, *dkey_out;  // score keys; afterwards the packed tp / fp and their scan
  int *didx_in, *didx_out;                 // detection indices; didx_in ends as the sorted permutation
  unsigned *ckey_in, *ckey_out;
  unsigned long long *gkey_in, *gkey_out;
  int *gidx_in, *gidx_out, *first_pos;
  long long *match, *cls_cnt;
  double* scratch;
  void* tmp;
  size_t tmp_bytes, total;
  EvalWs(void* base, long long n_det, long long n_gt, int nc) {
    Carver c(base);
    dkey_in = c.take<unsigned long long>(n_det);
    dkey_out = c.take<unsigned long long>(n_det);
    didx_in = c.take<int>(n_det);
    didx_out = c.take<int>(n_det);
    ckey_in = c.take<unsigned>(n_det);
    ckey_out = c.take<unsigned>(n_det);
    gkey_in = c.take<unsigned long long>(n_gt);
    gkey_out = c.take<unsigned long long>(n_gt);
    gidx_in = c.take<int>(n_gt);
    gidx_out = c.take<int>(n_gt);
    first_pos = c.take<int>(n_gt);
    match = c.take<long long>(n_det);
    cls_cnt = c.take<long long>(nc);
    scratch = c.take<double>((size_t)n_det + 2 * (size_t)nc);
    tmp_bytes = std::max(std::max(sort_pairs_bytes<unsigned long long>(n_det), sort_pairs_bytes<unsigned>(n_det)),
                         std::max(sort_pairs_bytes<unsigned long long>(n_gt), scan_bytes(n_det)));
    tmp = c.take<char>(tmp_bytes);
    total = c.used();
  }
};

unsigned blocks(long long n, int t) { return (unsigned)std::max<long long>(1, (n + t - 1) / t); }

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

size_t y5obb_dota_eval_workspace_bytes(int64_t n_det, int64_t n_gt, int n_images, int nc) {
  if (n_det < 0 || n_gt < 0 || n_images < 0 || nc <= 0) return 256;
  char probe;  // (only the offsets are used)
  EvalWs ws(&probe, n_det, n_gt, nc);
  return ws.total + 256;
}

int y5obb_dota_eval_f64(const int32_t* det_img, const double* det10, int64_t n_det, const int32_t* gt_img, const double* gt10,
                        int64_t n_gt, int n_images, int nc, double ovthresh, int use_07_metric, int64_t* class_off,
                        double* rec, double* prec, double* ap, int64_t* npos, int32_t* status, void* ws_ptr, size_t ws_bytes,
                        void* stream) {
  if (n_det < 0 || n_gt < 0 || n_images < 0 || nc <= 0 || n_det >= INT_MAX || n_gt >= INT_MAX || !class_off || !ap ||
      !npos || !status || !ws_ptr)
    return Y5OBB_EINVAL;
  if (n_det > 0 && (!det_img || !det10 || !rec || !prec)) return Y5OBB_EINVAL;
  if (n_gt > 0 && (!gt_img || !gt10)) return Y5OBB_EINVAL;
  if ((unsigned long long)nc * (unsigned long long)n_images >= (1ull << 62)) return Y5OBB_EINVAL;
  if (y5obb_dota_eval_workspace_bytes(n_det, n_gt, n_images, nc) > ws_bytes) return Y5OBB_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  EvalWs ws(ws_ptr, n_det, n_gt, nc);
  Y5_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  Y5_CUDA(cudaMemsetAsync(ws.cls_cnt, 0, sizeof(long long) * nc, st));
  Y5_CUDA(cudaMemsetAsync(npos, 0, sizeof(int64_t) * nc, st));
  size_t tmp = ws.tmp_bytes;
  // detections: descending score, then a stable pass by class -> per class in descending score, ties by input index
  if (n_det > 0) {
    k_eval_det_keys<<<blocks(n_det, 256), 256, 0, st>>>(det_img, det10, n_det, nc, n_images, ws.dkey_in, ws.didx_in,
                                                        ws.cls_cnt, status);
    Y5_LAUNCH_CHECK();
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.dkey_in, ws.dkey_out, ws.didx_in, ws.didx_out, (int)n_det, 0, 64,
                                            st));
    k_eval_cls_keys<<<blocks(n_det, 256), 256, 0, st>>>(det_img, det10, n_det, nc, n_images, ws.didx_out, ws.ckey_in);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.ckey_in, ws.ckey_out, ws.didx_out, ws.didx_in, (int)n_det, 0,
                                            bit_length((unsigned long long)nc), st));
  }
  k_eval_offsets<<<1, 1, 0, st>>>(ws.cls_cnt, nc, class_off);
  Y5_LAUNCH_CHECK();
  // ground truths grouped by (class, image), file order within a group
  if (n_gt > 0) {
    k_eval_gt_keys<<<blocks(n_gt, 256), 256, 0, st>>>(gt_img, gt10, n_gt, nc, n_images, ws.gkey_in, ws.gidx_in, npos,
                                                      ws.first_pos, status);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.gkey_in, ws.gkey_out, ws.gidx_in, ws.gidx_out, (int)n_gt, 0,
                                            bit_length((unsigned long long)nc * (unsigned long long)n_images), st));
  }
  if (n_det > 0) {
    k_eval_match<<<blocks(n_det, 128), 128, 0, st>>>(det_img, det10, n_det, gt10, ws.gkey_out, ws.gidx_out, n_gt, n_images,
                                                     ws.didx_in, class_off, nc, ovthresh, ws.match, ws.first_pos);
    Y5_LAUNCH_CHECK();
    k_eval_tpfp<<<blocks(n_det, 256), 256, 0, st>>>(ws.match, ws.first_pos, n_det, class_off, nc, ws.dkey_in);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceScan::InclusiveSum(ws.tmp, tmp, ws.dkey_in, ws.dkey_out, (int)n_det, st));
    k_eval_curve<<<blocks(n_det, 256), 256, 0, st>>>(ws.dkey_out, n_det, class_off, nc, npos, rec, prec);
    Y5_LAUNCH_CHECK();
  }
  k_eval_ap<<<nc, AP_THREADS, 0, st>>>(rec, prec, class_off, use_07_metric, ws.scratch, ap);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_task1_round_f64(const double* rows10, int64_t n, double* out10, void* stream) {
  if (n < 0 || (n > 0 && (!rows10 || !out10))) return Y5OBB_EINVAL;
  if (n == 0) return Y5OBB_OK;
  k_task1_round<<<blocks(n, 256), 256, 0, (cudaStream_t)stream>>>(rows10, n, out10);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
