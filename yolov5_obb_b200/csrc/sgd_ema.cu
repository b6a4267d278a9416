// Fused optimizer step + EMA update over all tensors of the model in ONE launch (SURVEY section 8f rank 1):
//   train.py:148-162,336-342   optimizer groups (BatchNorm weights / other weights with decay / biases), optimizer.step()
//   torch.optim.SGD(nesterov=True, dampening=0):  g' = g + wd * p;  buf = g' (first step) | momentum * buf + g';
//                                                 p -= lr * (g' + momentum * buf)
//   torch.optim.Adam (train.py --adam, train.py:157-163), torch's multi-tensor step with coupled L2 decay:
//                                                 g' = g + wd * p;  m = lerp(m, g', 1 - beta1);  v = beta2 * v + (1 - beta2) g'^2;
//                                                 p += step_size * m / (sqrt(v) / bc2_sqrt + eps)
//   utils/torch_utils.py:304-314                  ema = d * ema + (1 - d) * p  for every floating-point state_dict entry
// Every op is one _rn intrinsic rounded as torch rounds it, so parameters, momentum buffers, moments and EMA are bit-equal to
// torch.optim.SGD / torch.optim.Adam's foreach steps and ModelEMA.update's per-tensor ops (tests/test_sgd_exact_gpu.py,
// tests/test_adam_ema_gpu.py).  train_step.TrainStep uses it whenever every batch ends with an optimizer step (it replaces
// about 60 multi-tensor launches, 0.6 ms per yolov5m step).
// HBM-bound: SGD 16 B read + 12 B written per parameter element, Adam 20 B read + 16 B written.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace y5obb {
namespace {

struct SgdEntryK {
  float* p;
  const float* g;
  float* mom;
  float* ema;
  long long first;  // global index of this tensor's first element
  long long n;
  float weight_decay;
  int group;        // 0..2: index into the per-step lr table; -1: EMA only (buffers)
};

struct AdamEntryK {
  float* p;
  const float* g;
  float* exp_avg;
  float* exp_avg_sq;
  float* ema;
  long long first;  // global index of this tensor's first element
  long long n;
  float weight_decay;
  int group;        // 0..2: index into the per-step step-size table; -1: EMA only (buffers)
};

template <typename K>
struct TablePlan {
  K* table = nullptr;
  int n = 0;
  long long total = 0;
};

struct SgdStep {
  float lr[3];
  float momentum;
  float ema_d, ema_c;      // fp32(d) and fp32(1 - d), 1 - d formed in double
  int first_step;
};

struct AdamStep {
  float step_size[3];      // -lr / (1 - beta1^t) per group
  float lerp_w;            // 1 - beta1
  float beta2, one_minus_beta2;
  float bc2_sqrt, eps;
  float ema_d, ema_c;      // as SgdStep
};

// The entry that holds global element i (entries are ordered by `first`).
template <typename K>
__device__ __forceinline__ K find_entry(const K* __restrict__ table, int n, long long i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].first <= i) lo = mid; else hi = mid - 1;
  }
  return table[lo];
}

// ModelEMA.update for one element, as the reference's per-tensor ops round it on CUDA: v *= d (fp32(d)), then
// v += (1 - d) * p, where the product is its own rounded op with 1 - d formed in double and read as fp32.
__device__ __forceinline__ void ema_update(float* ema, long long j, float p, float d, float c) {
  if (ema) ema[j] = __fadd_rn(__fmul_rn(ema[j], d), __fmul_rn(c, p));
}

__global__ void k_sgd_ema(const SgdEntryK* __restrict__ table, int n, long long total, SgdStep s) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const SgdEntryK e = find_entry(table, n, i);
    const long long j = i - e.first;
    float p = e.p[j];
    if (e.group >= 0) {
      float g = e.g[j];
      if (e.weight_decay != 0.f) g = __fmaf_rn(e.weight_decay, p, g);                    // _foreach_add(grads, params, alpha=wd)
      const float buf = s.first_step ? g : __fadd_rn(__fmul_rn(e.mom[j], s.momentum), g); // _foreach_mul_(bufs, momentum);
      e.mom[j] = buf;                                                                      // _foreach_add_(bufs, grads)
      g = __fmaf_rn(s.momentum, buf, g);                                                   // _foreach_add_(grads, bufs, alpha=momentum)
      p = __fmaf_rn(-s.lr[e.group], g, p);                                                 // _foreach_add_(params, grads, alpha=-lr)
      e.p[j] = p;
    }
    ema_update(e.ema, j, p, s.ema_d, s.ema_c);
  }
}

// torch/optim/adam.py _multi_tensor_adam (foreach, capturable=False, amsgrad=False), one ATen foreach op per line, each rounded
// as the sm_90 SASS shipped with torch rounds it: the alpha add, lerp and addcmul / addcdiv scalars are fused multiply-adds,
// the two divisions and the square root are IEEE-rounded (no reciprocal multiply).
__global__ void k_adam_ema(const AdamEntryK* __restrict__ table, int n, long long total, AdamStep s) {
  const bool lerp_small = fabsf(s.lerp_w) < 0.5f;   // ATen's lerp: self + w (end - self) | end - (end - self)(1 - w)
  const float lerp_c = __fsub_rn(1.0f, s.lerp_w);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const AdamEntryK e = find_entry(table, n, i);
    const long long j = i - e.first;
    float p = e.p[j];
    if (e.group >= 0) {
      float g = e.g[j];
      if (e.weight_decay != 0.f) g = __fmaf_rn(e.weight_decay, p, g);                   // _foreach_add(grads, params, alpha=wd)
      float m = e.exp_avg[j];
      const float dm = __fsub_rn(g, m);
      m = lerp_small ? __fmaf_rn(dm, s.lerp_w, m) : __fmaf_rn(-lerp_c, dm, g);           // _foreach_lerp_(exp_avgs, grads, 1 - b1)
      float v = __fmul_rn(e.exp_avg_sq[j], s.beta2);                                     // _foreach_mul_(exp_avg_sqs, beta2)
      v = s.one_minus_beta2 == 1.0f ? __fmaf_rn(g, g, v)                                 // _foreach_addcmul_(.., g, g, 1 - b2)
                                    : __fmaf_rn(__fmul_rn(g, g), s.one_minus_beta2, v);
      e.exp_avg[j] = m;
      e.exp_avg_sq[j] = v;
      float d = __fsqrt_rn(v);                                                           // _foreach_sqrt(exp_avg_sqs)
      d = __fdiv_rn(d, s.bc2_sqrt);                                                      // _foreach_div_(.., bias_correction2_sqrt)
      d = __fadd_rn(d, s.eps);                                                           // _foreach_add_(.., eps)
      p = __fmaf_rn(__fdiv_rn(m, d), s.step_size[e.group], p);                           // _foreach_addcdiv_(params, m, d, step)
      e.p[j] = p;
    }
    ema_update(e.ema, j, p, s.ema_d, s.ema_c);
  }
}

template <typename K>
int upload_table(const std::vector<K>& h, long long total, TablePlan<K>** out) {
  TablePlan<K>* p = new TablePlan<K>();
  p->n = (int)h.size();
  p->total = total;
  cudaError_t err = cudaMalloc(&p->table, sizeof(K) * h.size());
  if (err == cudaSuccess) err = cudaMemcpy(p->table, h.data(), sizeof(K) * h.size(), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    if (p->table) cudaFree(p->table);
    delete p;
    return cuda_fail(err);
  }
  *out = p;
  return Y5OBB_OK;
}

template <typename K>
void destroy_table(TablePlan<K>* p) {
  if (!p) return;
  if (p->table) cudaFree(p->table);
  delete p;
}

template <typename K>
int grid_for(const TablePlan<K>* p) {
  return (int)std::min<long long>((p->total + 255) / 256, (long long)sm_count() * 32);
}

using SgdPlan = TablePlan<SgdEntryK>;
using AdamPlan = TablePlan<AdamEntryK>;

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_sgd_ema_plan_create(const y5obb_sgd_entry* entries, int n, y5obb_sgd_plan_t** out) {
  if (!entries || n <= 0 || !out) return Y5OBB_EINVAL;
  std::vector<SgdEntryK> h((size_t)n);
  long long total = 0;
  for (int i = 0; i < n; ++i) {
    const y5obb_sgd_entry& e = entries[i];
    if (!e.p || e.n <= 0 || e.group < -1 || e.group > 2) return Y5OBB_EINVAL;
    if (e.group >= 0 && (!e.g || !e.mom)) return Y5OBB_EINVAL;
    if (e.group < 0 && !e.ema) return Y5OBB_EINVAL;  // an EMA-only entry without an EMA does nothing: a malformed table
    SgdEntryK& k = h[(size_t)i];
    k.p = e.p;
    k.g = e.g;
    k.mom = e.mom;
    k.ema = e.ema;
    k.first = total;
    k.n = e.n;
    k.weight_decay = e.weight_decay;
    k.group = e.group;
    total += e.n;
  }
  SgdPlan* p = nullptr;
  const int rc = upload_table(h, total, &p);
  if (rc == Y5OBB_OK) *out = reinterpret_cast<y5obb_sgd_plan_t*>(p);
  return rc;
}

int y5obb_sgd_ema_plan_run(const y5obb_sgd_plan_t* plan, const float* lr3, float momentum, double ema_decay, int first_step,
                           void* stream) {
  if (!plan || !lr3 || !(momentum >= 0.f) || !(ema_decay >= 0.0 && ema_decay <= 1.0)) return Y5OBB_EINVAL;
  const SgdPlan* p = reinterpret_cast<const SgdPlan*>(plan);
  SgdStep s;
  s.lr[0] = lr3[0];
  s.lr[1] = lr3[1];
  s.lr[2] = lr3[2];
  s.momentum = momentum;
  s.ema_d = (float)ema_decay;
  s.ema_c = (float)(1.0 - ema_decay);      // ModelEMA: (1 - d) * msd[k], a Python float read as fp32
  s.first_step = first_step;
  k_sgd_ema<<<grid_for(p), 256, 0, (cudaStream_t)stream>>>(p->table, p->n, p->total, s);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

void y5obb_sgd_ema_plan_destroy(y5obb_sgd_plan_t* plan) { destroy_table(reinterpret_cast<SgdPlan*>(plan)); }

int y5obb_adam_ema_plan_create(const y5obb_adam_entry* entries, int n, y5obb_adam_plan_t** out) {
  if (!entries || n <= 0 || !out) return Y5OBB_EINVAL;
  std::vector<AdamEntryK> h((size_t)n);
  long long total = 0;
  for (int i = 0; i < n; ++i) {
    const y5obb_adam_entry& e = entries[i];
    if (!e.p || e.n <= 0 || e.group < -1 || e.group > 2) return Y5OBB_EINVAL;
    if (e.group >= 0 && (!e.g || !e.exp_avg || !e.exp_avg_sq)) return Y5OBB_EINVAL;
    if (e.group < 0 && !e.ema) return Y5OBB_EINVAL;  // an EMA-only entry without an EMA does nothing: a malformed table
    AdamEntryK& k = h[(size_t)i];
    k.p = e.p;
    k.g = e.g;
    k.exp_avg = e.exp_avg;
    k.exp_avg_sq = e.exp_avg_sq;
    k.ema = e.ema;
    k.first = total;
    k.n = e.n;
    k.weight_decay = e.weight_decay;
    k.group = e.group;
    total += e.n;
  }
  AdamPlan* p = nullptr;
  const int rc = upload_table(h, total, &p);
  if (rc == Y5OBB_OK) *out = reinterpret_cast<y5obb_adam_plan_t*>(p);
  return rc;
}

int y5obb_adam_ema_plan_run(const y5obb_adam_plan_t* plan, const float* step_size3, double beta1, double beta2,
                            float bc2_sqrt, float eps, double ema_decay, void* stream) {
  if (!plan || !step_size3) return Y5OBB_EINVAL;
  if (!(beta1 >= 0.0 && beta1 < 1.0) || !(beta2 >= 0.0 && beta2 < 1.0) || !(bc2_sqrt > 0.f)) return Y5OBB_EINVAL;
  if (!(ema_decay >= 0.0 && ema_decay <= 1.0)) return Y5OBB_EINVAL;
  const AdamPlan* p = reinterpret_cast<const AdamPlan*>(plan);
  AdamStep s;
  s.step_size[0] = step_size3[0];
  s.step_size[1] = step_size3[1];
  s.step_size[2] = step_size3[2];
  s.lerp_w = (float)(1.0 - beta1);          // torch: _foreach_lerp_(.., 1 - beta1), a Python float read as float
  s.beta2 = (float)beta2;
  s.one_minus_beta2 = (float)(1.0 - beta2);
  s.bc2_sqrt = bc2_sqrt;
  s.eps = eps;
  s.ema_d = (float)ema_decay;
  s.ema_c = (float)(1.0 - ema_decay);
  k_adam_ema<<<grid_for(p), 256, 0, (cudaStream_t)stream>>>(p->table, p->n, p->total, s);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

void y5obb_adam_ema_plan_destroy(y5obb_adam_plan_t* plan) { destroy_table(reinterpret_cast<AdamPlan*>(plan)); }

}  // extern "C"
