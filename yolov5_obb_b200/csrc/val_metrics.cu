// Validation metrics on the device: the stats accumulation of val.py:209-250, then utils/metrics.py:21-114 ap_per_class
// (plot=False) with compute_ap, bit for bit in fp64.
//   y5obb_val_stats_append   one launch per batch: the valid NMS rows (tp[niou], conf, cls) and their (image, row) position
//                            appended at a running row count kept on the device, the labels' classes added to nt [nc].
//   y5obb_ap_per_class_f64   ap [n_u, niou], p / r [n_u, 1000] and the classes with labels, without a host read.
//
// ap_per_class pipeline over the whole buffer capacity (rows at or past *n_rows carry sentinel keys and sort behind every
// class, so the host never reads the row count): [CUB radix sort by (image, row) when rows were appended out of order] ->
// stable radix sort by descending conf -> stable radix sort by class (classes without labels go to a bucket past the last
// class) -> k_vm_gather (tp columns in sorted order, [niou][N]) -> CUB inclusive scan = exact integer tpc per class and
// column -> k_vm_curves (recall, precision; precision written reversed with its (column, class) segment key) -> CUB
// InclusiveScanByKey with max = the suffix-max envelope of every (class, column) at once -> k_vm_grid (the 1000-point p / r
// curves, np.interp) -> k_vm_ap (compute_ap's 101-point np.interp and np.trapz, one block per (class, column)).
//
// Every fp64 step is a separately rounded __d*_rn op in numpy's order (no FMA contraction).  The 101-point interpolation of
// compute_ap assumes recall <= 1 in every column (each label claims at most one detection, as y5obb_val_match_f32 decides):
// then [0, recall, 1] is non-decreasing and "the last index j with xp[j] <= x" is what numpy's binary search finds.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cub/cub.cuh>

#include "common.cuh"
#include "np_sum.cuh"

namespace y5obb {
namespace {

constexpr int VS_STATUS_CLASS = 1, VS_STATUS_CAPACITY = 2;
constexpr int VS_THREADS = 256;
constexpr int VS_MAX_BATCH = 4096;
constexpr int GRID_N = 1000;  // px = np.linspace(0, 1, 1000)
constexpr int AP_N = 101;     // x = np.linspace(0, 1, 101)

struct AppendArgs {
  const float* pred7;       // [B, max_det, 7] (cx, cy, l, s, theta, conf, cls)
  const long long* counts;  // [B] rows per image (+ [B] = total candidates when nms_cap >= 0)
  int B, max_det;
  long long nms_cap;        // < 0: no capacity check
  const uint8_t* correct;   // [B, max_det, niou]
  int niou;
  const float* labels;      // [nl, label_stride] (image, cls, ...)
  long long nl;
  int label_stride;
  long long image_base;
  uint8_t* tp;              // [capacity, niou]
  float* conf;
  int32_t* cls;
  long long* key;           // (image << 32) | row
  long long capacity;
  long long* n_rows;
  unsigned long long* nt;   // [nc]
  int nc;
  int32_t* flags;           // [0] status bits, [1] some tp byte set, [2] finished-block counter (0 between launches)
  int32_t* skip;
};

__device__ __forceinline__ bool valid_class(float c, int nc) { return c >= 0.f && c < (float)nc && c == floorf(c); }

__global__ void __launch_bounds__(VS_THREADS) k_vs_append(AppendArgs a) {
  extern __shared__ long long s_off[];  // [B + 1] exclusive prefix of the valid rows per image
  __shared__ long long s_base;
  __shared__ int s_bad;
  if (threadIdx.x == 0) {
    bool bad = false;
    if (a.nms_cap >= 0) {
      const long long tot = a.counts[a.B];
      bad = tot > a.nms_cap || tot < 0;
      for (int b = 0; b < a.B; ++b) bad = bad || a.counts[b] < 0;
    }
    long long s = 0;
    for (int b = 0; b < a.B; ++b) {
      s_off[b] = s;
      s += bad ? 0 : min((long long)a.max_det, max(0ll, a.counts[b]));
    }
    s_off[a.B] = s;
    s_bad = bad;
    s_base = *(volatile long long*)a.n_rows;
  }
  __syncthreads();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nrow = (long long)a.B * a.max_det;
  if (!s_bad && t < nrow) {
    const int b = (int)(t / a.max_det), r = (int)(t % a.max_det);
    if (s_off[b] + r < s_off[b + 1]) {
      const long long dst = s_base + s_off[b] + r;
      if (dst >= a.capacity) {
        atomicOr(a.flags, VS_STATUS_CAPACITY);
      } else {
        const uint8_t* c = a.correct + t * a.niou;
        uint8_t* o = a.tp + dst * a.niou;
        int any = 0;
        for (int k = 0; k < a.niou; ++k) {
          const uint8_t v = c[k] != 0;
          o[k] = v;
          any |= v;
        }
        if (any) a.flags[1] = 1;
        const float* P = a.pred7 + t * 7;
        a.conf[dst] = P[5];
        const bool ok = valid_class(P[6], a.nc);
        if (!ok) atomicOr(a.flags, VS_STATUS_CLASS);
        a.cls[dst] = ok ? (int32_t)P[6] : -1;
        a.key[dst] = ((a.image_base + b) << 32) | (long long)r;
      }
    }
  } else if (!s_bad && t < nrow + a.nl) {
    // val.py:214 takes the labels of images 0 .. nb - 1; other rows belong to no image of the batch
    const float* L = a.labels + (t - nrow) * a.label_stride;
    const float img = L[0];
    if (img >= 0.f && img < (float)a.B && img == floorf(img)) {
      if (valid_class(L[1], a.nc)) atomicAdd(a.nt + (int)L[1], 1ull);
      else atomicOr(a.flags, VS_STATUS_CLASS);
    }
  }
  // the last block to finish moves the running row count (every block has read it by then) and reports the skip
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(reinterpret_cast<unsigned*>(a.flags + 2), 1u);
    if (prev == gridDim.x - 1) {
      __threadfence();
      *a.n_rows = s_base + s_off[a.B];
      *a.skip = s_bad;
      a.flags[2] = 0;
    }
  }
}

// ascending order of the key = descending conf (argsort of -conf); -0.0 ties with +0.0, NaN after every number
__device__ __forceinline__ unsigned desc_conf_key(float c) {
  if (isnan(c)) return 0xfffffffeu;
  const unsigned b = __float_as_uint(__fadd_rn(c, 0.0f));
  const unsigned asc = (b >> 31) ? ~b : (b | 0x80000000u);
  return ~asc;
}

__device__ __forceinline__ long long valid_rows(const long long* n_rows, long long capacity) {
  return min(*n_rows, capacity);
}

__global__ void k_vm_pos_keys(const long long* __restrict__ key, const long long* __restrict__ n_rows, long long N,
                              unsigned long long* __restrict__ pos_key, int* __restrict__ idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  idx[i] = (int)i;
  if (pos_key) pos_key[i] = i < valid_rows(n_rows, N) ? (unsigned long long)key[i] : ~0ull;
}

__global__ void k_vm_conf_keys(const float* __restrict__ conf, const long long* __restrict__ n_rows, long long N,
                               const int* __restrict__ perm, unsigned* __restrict__ ckey) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const int i = perm[p];
  ckey[p] = i < valid_rows(n_rows, N) ? desc_conf_key(conf[i]) : 0xffffffffu;
}

// class of each conf-sorted row; nc for rows past the count and for classes without labels (ap_per_class skips them)
__global__ void k_vm_cls_keys(const int32_t* __restrict__ cls, const long long* __restrict__ n_rows, long long N,
                              const int* __restrict__ perm, const unsigned long long* __restrict__ nt, int nc,
                              unsigned* __restrict__ ckey, unsigned long long* __restrict__ cls_cnt) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const int i = perm[p];
  int c = i < valid_rows(n_rows, N) ? cls[i] : nc;
  if (c < 0 || c >= nc || nt[c] == 0) c = nc;
  ckey[p] = (unsigned)c;
  if (c < nc) atomicAdd(cls_cnt + c, 1ull);
}

// class_off [nc + 1] and np.unique(target_cls): the classes with labels, ascending
__global__ void k_vm_offsets(const unsigned long long* __restrict__ cls_cnt, const unsigned long long* __restrict__ nt, int nc,
                             long long* __restrict__ off, int32_t* __restrict__ ap_class, int32_t* __restrict__ n_u) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  long long s = 0;
  int u = 0;
  off[0] = 0;
  for (int c = 0; c < nc; ++c) {
    off[c + 1] = (s += (long long)cls_cnt[c]);
    if (nt[c] > 0) ap_class[u++] = c;
  }
  *n_u = u;
  for (int k = u; k < nc; ++k) ap_class[k] = -1;
}

// tp columns in sorted order ([niou][N], 0 past the class rows) and the sorted confidences
__global__ void k_vm_gather(const uint8_t* __restrict__ tp, const float* __restrict__ conf, const int* __restrict__ perm,
                            const long long* __restrict__ off, int nc, int niou, long long N, unsigned* __restrict__ tpf,
                            float* __restrict__ conf_s) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const bool in = p < off[nc];
  const int i = perm[p];
  for (int j = 0; j < niou; ++j) tpf[(long long)j * N + p] = in ? (unsigned)tp[(long long)i * niou + j] : 0u;
  conf_s[p] = in ? conf[i] : 0.f;
}

__device__ __forceinline__ int class_of(const long long* off, int nc, long long p) {  // largest c with off[c] <= p
  int lo = 0, hi = nc - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= p) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// recall = tpc / (n_l + eps), precision = tpc / (tpc + fpc) (fpc = position - tpc); precision and the (column, class)
// segment key are written at the mirrored index so that a forward scan by key is the reverse (suffix) max
__global__ void k_vm_curves(const unsigned* __restrict__ csum, const long long* __restrict__ off, int nc,
                            const unsigned long long* __restrict__ nt, long long N, long long M, double* __restrict__ recall,
                            double* __restrict__ prec_rev, unsigned* __restrict__ key_rev) {
  const long long f = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= M) return;
  const long long j = f / N, p = f - j * N, q = M - 1 - f;
  if (p >= off[nc]) {
    recall[f] = 0.0;
    prec_rev[q] = 0.0;
    key_rev[q] = (unsigned)(j * (nc + 1) + nc);
    return;
  }
  const int c = class_of(off, nc, p);
  const long long s = off[c], fs = j * N + s;
  const double tpc = (double)(csum[f] - (fs > 0 ? csum[fs - 1] : 0u));
  recall[f] = __ddiv_rn(tpc, __dadd_rn((double)nt[c], 1e-16));
  prec_rev[q] = __ddiv_rn(tpc, (double)(p - s + 1));
  key_rev[q] = (unsigned)(j * (nc + 1) + c);
}

struct NpMax {  // np.maximum: NaN propagates
  __device__ __forceinline__ double operator()(const double& a, const double& b) const {
    return (a > b || isnan(a)) ? a : b;
  }
};

// np.interp(x, xp, fp, left, right = fp[-1]) (numpy/_core/src/multiarray/compiled_base.c arr_interp) on a non-decreasing xp
// of n points given by accessors.  The slope expression, the exact-hit rule and the NaN fallback are numpy's.
template <class XP, class FP>
__device__ double np_interp(double x, long long n, XP xp, FP fp, double left) {
  const double right = fp(n - 1);
  if (isnan(x)) return x;
  if (n == 1) {
    const double x0 = xp(0);
    return x < x0 ? left : (x > x0 ? right : fp(0));
  }
  long long lo = 0, hi = n;  // j = the last index with xp[j] <= x, -1 when x < xp[0]
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (xp(mid) <= x) lo = mid + 1; else hi = mid;
  }
  const long long j = lo - 1;
  if (j < 0) return left;
  if (j >= n - 1) return right;
  const double xj = xp(j);
  if (xj == x) return fp(j);
  const double x1 = xp(j + 1), fj = fp(j), f1 = fp(j + 1);
  const double slope = __ddiv_rn(__dsub_rn(f1, fj), __dsub_rn(x1, xj));
  double res = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xj)), fj);
  if (isnan(res)) {
    res = __dadd_rn(__dmul_rn(slope, __dsub_rn(x, x1)), f1);
    if (isnan(res) && fj == f1) res = fj;
  }
  return res;
}

// np.linspace(0, 1, num): k * (1 / (num - 1)), the last point 1.0
__device__ __forceinline__ double np_linspace01(int k, int num) {
  return k == num - 1 ? 1.0 : __dmul_rn((double)k, __ddiv_rn(1.0, (double)(num - 1)));
}

// r[u] = np.interp(-px, -conf, recall[:, 0], left=0), p[u] = np.interp(-px, -conf, precision[:, 0], left=1)
__global__ void k_vm_grid(const long long* __restrict__ off, const int32_t* __restrict__ ap_class,
                          const int32_t* __restrict__ n_u, int nc, const float* __restrict__ conf_s,
                          const double* __restrict__ recall, const double* __restrict__ prec_rev, long long M,
                          double* __restrict__ p_out, double* __restrict__ r_out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)nc * GRID_N) return;
  const int u = (int)(t / GRID_N), k = (int)(t % GRID_N);
  double pv = 0.0, rv = 0.0;
  if (u < *n_u) {
    const int c = ap_class[u];
    const long long s = off[c], n = off[c + 1] - s;
    if (n > 0) {
      const double x = -np_linspace01(k, GRID_N);
      auto xp = [=](long long i) { return -(double)conf_s[s + i]; };
      rv = np_interp(x, n, xp, [=](long long i) { return recall[s + i]; }, 0.0);
      pv = np_interp(x, n, xp, [=](long long i) { return prec_rev[M - 1 - (s + i)]; }, 1.0);
    }
  }
  p_out[t] = pv;
  r_out[t] = rv;
}

constexpr int AP_THREADS = 128;

// compute_ap(recall[:, j], precision[:, j]): mrec = [0, recall, 1], mpre = the envelope of [1, precision, 0],
// ap = np.trapz(np.interp(x, mrec, mpre), x) with x = np.linspace(0, 1, 101); one block per (class, column)
__global__ void __launch_bounds__(AP_THREADS) k_vm_ap(const long long* __restrict__ off, const int32_t* __restrict__ ap_class,
                                                      const int32_t* __restrict__ n_u, int niou, long long N, long long M,
                                                      const double* __restrict__ recall, const double* __restrict__ env_rev,
                                                      double* __restrict__ ap) {
  __shared__ double s_x[AP_N], s_y[AP_N], s_t[AP_N - 1];
  const int u = blockIdx.x, j = blockIdx.y;
  long long s = 0, n = 0;
  if (u < *n_u) {
    const int c = ap_class[u];
    s = off[c];
    n = off[c + 1] - s;
  }
  if (n == 0) {
    if (threadIdx.x == 0) ap[(long long)u * niou + j] = 0.0;
    return;
  }
  const long long base = (long long)j * N + s;
  auto env = [=](long long i) { return env_rev[M - 1 - (base + i)]; };  // suffix max of precision[i:] in the segment
  auto mrec = [=](long long i) { return i == 0 ? 0.0 : (i <= n ? recall[base + i - 1] : 1.0); };
  NpMax mx;
  auto mpre = [=](long long i) { return i == 0 ? mx(mx(0.0, env(0)), 1.0) : (i <= n ? mx(0.0, env(i - 1)) : 0.0); };
  for (int k = threadIdx.x; k < AP_N; k += AP_THREADS) {
    const double x = np_linspace01(k, AP_N);
    s_x[k] = x;
    s_y[k] = np_interp(x, n + 2, mrec, mpre, mpre(0));
  }
  __syncthreads();
  for (int k = threadIdx.x; k < AP_N - 1; k += AP_THREADS)  // diff(x) * (y[1:] + y[:-1]) / 2.0
    s_t[k] = __ddiv_rn(__dmul_rn(__dsub_rn(s_x[k + 1], s_x[k]), __dadd_rn(s_y[k + 1], s_y[k])), 2.0);
  __syncthreads();
  if (threadIdx.x == 0) ap[(long long)u * niou + j] = np_pairwise_sum(s_t, AP_N - 1);
}

__global__ void k_vm_fill_ap(int nc, int niou, double* __restrict__ ap) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nc * niou) ap[t] = 0.0;
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

size_t scan_bytes(long long m) {
  size_t b = 0, c = 0;
  if (m <= 0) return 0;
  if (cub::DeviceScan::InclusiveSum(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (int)m) != cudaSuccess ||
      cub::DeviceScan::InclusiveScanByKey(nullptr, c, (const unsigned*)nullptr, (const double*)nullptr, (double*)nullptr,
                                          NpMax(), (int)m) != cudaSuccess) {
    (void)cudaGetLastError();
    return (size_t)(32u << 20) + (size_t)m * 16;
  }
  return std::max(b, c);
}

struct ApWs {
  unsigned long long *pos_in, *pos_out, *cls_cnt;
  int *idx_a, *idx_b;
  unsigned *ck_in, *ck_out, *tpf, *csum;
  long long* off;
  float* conf_s;
  double *recall, *prec_rev, *env_rev;
  void* tmp;
  size_t tmp_bytes, total;
  ApWs(void* base, long long N, int niou, int nc) {
    const long long M = N * niou;
    Carver c(base);
    pos_in = c.take<unsigned long long>(N);
    pos_out = c.take<unsigned long long>(N);
    cls_cnt = c.take<unsigned long long>(nc);
    idx_a = c.take<int>(N);
    idx_b = c.take<int>(N);
    ck_in = c.take<unsigned>(N);
    ck_out = c.take<unsigned>(N);
    tpf = c.take<unsigned>(M);
    csum = c.take<unsigned>(M);
    off = c.take<long long>(nc + 1);
    conf_s = c.take<float>(N);
    recall = c.take<double>(M);
    prec_rev = c.take<double>(M);
    env_rev = c.take<double>(M);
    tmp_bytes = std::max(std::max(sort_pairs_bytes<unsigned long long>(N), sort_pairs_bytes<unsigned>(N)), scan_bytes(M));
    tmp = c.take<char>(tmp_bytes);
    total = c.used();
  }
};

unsigned blocks(long long n, int t) { return (unsigned)std::max<long long>(1, (n + t - 1) / t); }

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_val_stats_append(const float* pred7, const int64_t* counts, int batch, int max_det, int64_t nms_cap,
                           const uint8_t* correct, int niou, const float* labels, int64_t n_labels, int label_stride,
                           int64_t image_base, uint8_t* tp, float* conf, int32_t* cls, int64_t* key, int64_t capacity,
                           int64_t* n_rows, int64_t* nt, int nc, int32_t* flags, int32_t* skip, void* stream) {
  if (batch <= 0 || batch > VS_MAX_BATCH || max_det <= 0 || niou <= 0 || n_labels < 0 || label_stride < 2 || nc <= 0 ||
      capacity < 0 || image_base < 0 || image_base + batch > INT_MAX)
    return Y5OBB_EINVAL;
  if (!pred7 || !counts || !correct || (n_labels > 0 && !labels) || !n_rows || !nt || !flags || !skip ||
      (capacity > 0 && (!tp || !conf || !cls || !key)))
    return Y5OBB_EINVAL;
  AppendArgs a;
  a.pred7 = pred7;
  a.counts = reinterpret_cast<const long long*>(counts);
  a.B = batch;
  a.max_det = max_det;
  a.nms_cap = nms_cap;
  a.correct = correct;
  a.niou = niou;
  a.labels = labels;
  a.nl = n_labels;
  a.label_stride = label_stride;
  a.image_base = image_base;
  a.tp = tp;
  a.conf = conf;
  a.cls = cls;
  a.key = reinterpret_cast<long long*>(key);
  a.capacity = capacity;
  a.n_rows = reinterpret_cast<long long*>(n_rows);
  a.nt = reinterpret_cast<unsigned long long*>(nt);
  a.nc = nc;
  a.flags = flags;
  a.skip = skip;
  const long long work = (long long)batch * max_det + n_labels;
  k_vs_append<<<blocks(work, VS_THREADS), VS_THREADS, sizeof(long long) * (batch + 1), (cudaStream_t)stream>>>(a);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

size_t y5obb_ap_per_class_workspace_bytes(int64_t capacity, int niou, int nc) {
  if (capacity < 0 || niou <= 0 || nc <= 0) return 256;
  char probe;  // (only the offsets are used)
  ApWs ws(&probe, capacity, niou, nc);
  return ws.total + 256;
}

int y5obb_ap_per_class_f64(const uint8_t* tp, const float* conf, const int32_t* cls, const int64_t* key, const int64_t* n_rows,
                           int64_t capacity, int ordered, const int64_t* nt, int nc, int niou, double* ap, double* p, double* r,
                           int32_t* ap_class, int32_t* n_u, void* ws_ptr, size_t ws_bytes, void* stream) {
  if (capacity < 0 || niou <= 0 || nc <= 0 || (long long)capacity * niou > INT_MAX || (long long)nc * (niou + 1) > INT_MAX)
    return Y5OBB_EINVAL;
  if (!n_rows || !nt || !ap || !p || !r || !ap_class || !n_u || !ws_ptr) return Y5OBB_EINVAL;
  if (capacity > 0 && (!tp || !conf || !cls || !key)) return Y5OBB_EINVAL;
  if (y5obb_ap_per_class_workspace_bytes(capacity, niou, nc) > ws_bytes) return Y5OBB_EWORKSPACE;
  cudaStream_t st = (cudaStream_t)stream;
  const long long N = capacity, M = N * niou;
  const long long* nr = reinterpret_cast<const long long*>(n_rows);
  const unsigned long long* ntu = reinterpret_cast<const unsigned long long*>(nt);
  ApWs ws(ws_ptr, N, niou, nc);
  Y5_CUDA(cudaMemsetAsync(ws.cls_cnt, 0, sizeof(unsigned long long) * nc, st));
  int* perm = ws.idx_a;
  if (N > 0) {
    size_t tmp = ws.tmp_bytes;
    k_vm_pos_keys<<<blocks(N, 256), 256, 0, st>>>(reinterpret_cast<const long long*>(key), nr, N, ordered ? nullptr : ws.pos_in,
                                                  ws.idx_a);
    Y5_LAUNCH_CHECK();
    if (!ordered) {  // rows appended out of order (a batch re-run after an NMS overflow): (image, row) order first
      Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.pos_in, ws.pos_out, ws.idx_a, ws.idx_b, (int)N, 0, 64, st));
      perm = ws.idx_b;
    }
    int* other = perm == ws.idx_a ? ws.idx_b : ws.idx_a;
    k_vm_conf_keys<<<blocks(N, 256), 256, 0, st>>>(conf, nr, N, perm, ws.ck_in);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.ck_in, ws.ck_out, perm, other, (int)N, 0, 32, st));
    std::swap(perm, other);
    k_vm_cls_keys<<<blocks(N, 256), 256, 0, st>>>(cls, nr, N, perm, ntu, nc, ws.ck_in, ws.cls_cnt);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceRadixSort::SortPairs(ws.tmp, tmp, ws.ck_in, ws.ck_out, perm, other, (int)N, 0,
                                            bit_length((unsigned long long)nc), st));
    std::swap(perm, other);
  }
  k_vm_offsets<<<1, 1, 0, st>>>(ws.cls_cnt, ntu, nc, ws.off, ap_class, n_u);
  Y5_LAUNCH_CHECK();
  if (N > 0) {
    k_vm_gather<<<blocks(N, 256), 256, 0, st>>>(tp, conf, perm, ws.off, nc, niou, N, ws.tpf, ws.conf_s);
    Y5_LAUNCH_CHECK();
    size_t tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceScan::InclusiveSum(ws.tmp, tmp, ws.tpf, ws.csum, (int)M, st));
    k_vm_curves<<<blocks(M, 256), 256, 0, st>>>(ws.csum, ws.off, nc, ntu, N, M, ws.recall, ws.prec_rev, ws.tpf);
    Y5_LAUNCH_CHECK();
    tmp = ws.tmp_bytes;
    Y5_CUDA(cub::DeviceScan::InclusiveScanByKey(ws.tmp, tmp, ws.tpf, ws.prec_rev, ws.env_rev, NpMax(), (int)M,
                                                cub::Equality(), st));
  }
  k_vm_grid<<<blocks((long long)nc * GRID_N, 256), 256, 0, st>>>(ws.off, ap_class, n_u, nc, ws.conf_s, ws.recall, ws.prec_rev,
                                                                 M, p, r);
  Y5_LAUNCH_CHECK();
  if (N > 0) {
    k_vm_ap<<<dim3((unsigned)nc, (unsigned)niou), AP_THREADS, 0, st>>>(ws.off, ap_class, n_u, niou, N, M, ws.recall,
                                                                      ws.env_rev, ap);
  } else {
    k_vm_fill_ap<<<blocks((long long)nc * niou, 256), 256, 0, st>>>(nc, niou, ap);
  }
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
