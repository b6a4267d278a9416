// Re-packing of the fp32 master weights into the bf16 operand layouts of the tensor-core kernels, all layers in ONE
// launch.  Training updates the parameters every step (train.py:336), so the packed copies the TMA descriptors point at
// must be refreshed every step: forward layout [tap][cout_pad][cin_pad] (K-major B operand of conv_sm90.cu) and the
// data-gradient layout (the same kernel run with the weights transposed and the taps flipped).
// One thread per packed element; a table of entries (device resident, built once per plan) tells it where the element
// comes from.  HBM-bound: 4 B read + 2 B written per packed element.
#include <cuda_bf16.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace y5obb {
namespace {

struct PackEntryK {
  const float* src;
  void* dst;
  long long first;   // index of this entry's first packed element in the global numbering
  int kind, Cout, Cin, KH, KW, rows_pad, cols_pad, g_real, g_pad;
};

struct PackPlan {
  PackEntryK* table = nullptr;
  int n = 0;
  long long total = 0;
};

// packed element (tap, row, col) of an entry -> value
__device__ __forceinline__ float pack_value(const PackEntryK& e, int tap, int row, int col) {
  const int kh = tap / e.KW, kw = tap - kh * e.KW;
  switch (e.kind) {
    case Y5OBB_PACK_FWD: {  // row = co, col = ci
      if (row >= e.Cout || col >= e.Cin) return 0.f;
      return e.src[(((long long)row * e.Cin + col) * e.KH + kh) * e.KW + kw];
    }
    case Y5OBB_PACK_DGRAD: {  // the dgrad conv has Cout' = Cin, Cin' = Cout: row = ci, col = co, taps flipped
      if (row >= e.Cin || col >= e.Cout) return 0.f;
      return e.src[(((long long)col * e.Cin + row) * e.KH + (e.KH - 1 - kh)) * e.KW + (e.KW - 1 - kw)];
    }
    case Y5OBB_PACK_DGRAD_S2: {  // tap = th * KW' + tw of the parity class (ph, pw) = (g_real >> 1, g_real & 1)
      if (row >= e.Cin || col >= e.Cout) return 0.f;
      const int ph = e.g_real >> 1, pw = e.g_real & 1;
      const int kwp = pw ? 2 : 1;
      const int th = tap / kwp, tw = tap - th * kwp;
      const int skh = ph ? (th == 0 ? 2 : 0) : 1, skw = pw ? (tw == 0 ? 2 : 0) : 1;
      return e.src[(((long long)col * e.Cin + row) * e.KH + skh) * e.KW + skw];
    }
    case Y5OBB_PACK_STEM: {  // 6x6/s2 stem as a 3x1 conv over the 48-channel window of the space-to-depth image
      // tap = ty (KH = 3, KW = 1 here), col = tx * 16 + (dy * 2 + dx) * 3 + c -> w[row][c][2ty+dy][2tx+dx]
      if (row >= e.Cout || col >= 48) return 0.f;
      const int tx = col >> 4, ch = col & 15;
      if (ch >= 12) return 0.f;
      const int ph = ch / 3, c = ch - ph * 3, dy = ph >> 1, dx = ph & 1;
      return e.src[(((long long)row * 3 + c) * 6 + (2 * tap + dy)) * 6 + (2 * tx + dx)];
    }
    case Y5OBB_PACK_DETECT: {  // anchor a's g_real rows sit at [a * g_pad, a * g_pad + g_real)
      const int a = row / e.g_pad, r = row - a * e.g_pad;
      if (r >= e.g_real || col >= e.Cin) return 0.f;
      const int co = a * e.g_real + r;
      if (co >= e.Cout) return 0.f;
      return e.src[(long long)co * e.Cin + col];
    }
    case Y5OBB_PACK_DETECT_DGRAD: {  // row = ci, col = a * g_pad + r
      const int a = col / e.g_pad, r = col - a * e.g_pad;
      if (r >= e.g_real || row >= e.Cin) return 0.f;
      const int co = a * e.g_real + r;
      if (co >= e.Cout) return 0.f;
      return e.src[(long long)co * e.Cin + row];
    }
    default: {  // Y5OBB_PACK_DETECT_BIAS: fp32 vector, col = a * g_pad + r
      const int a = col / e.g_pad, r = col - a * e.g_pad;
      const int co = a * e.g_real + r;
      return (r < e.g_real && co < e.Cout) ? e.src[co] : 0.f;
    }
  }
}

__global__ void k_pack_weights(const PackEntryK* __restrict__ table, int n, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n - 1;  // last entry with first <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (table[mid].first <= i) lo = mid; else hi = mid - 1;
    }
    const PackEntryK e = table[lo];
    const long long j = i - e.first;
    const long long per_tap = (long long)e.rows_pad * e.cols_pad;
    const int tap = (int)(j / per_tap);
    const long long r = j - (long long)tap * per_tap;
    const int row = (int)(r / e.cols_pad), col = (int)(r - (long long)row * e.cols_pad);
    const float v = pack_value(e, tap, row, col);
    if (e.kind == Y5OBB_PACK_DETECT_BIAS) static_cast<float*>(e.dst)[j] = v;
    else static_cast<__nv_bfloat16*>(e.dst)[j] = __float2bfloat16(v);
  }
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_pack_plan_create(const y5obb_pack_entry* entries, int n, y5obb_pack_plan_t** out) {
  if (!entries || n <= 0 || !out) return Y5OBB_EINVAL;
  std::vector<PackEntryK> h((size_t)n);
  long long total = 0;
  for (int i = 0; i < n; ++i) {
    const y5obb_pack_entry& e = entries[i];
    if (!e.src || !e.dst || e.Cout <= 0 || e.Cin <= 0 || e.KH <= 0 || e.KW <= 0 || e.rows_pad <= 0 || e.cols_pad <= 0 ||
        e.kind < Y5OBB_PACK_FWD || e.kind > Y5OBB_PACK_DGRAD_S2)
      return Y5OBB_EINVAL;
    if (e.kind == Y5OBB_PACK_DGRAD_S2 && (e.KH != 3 || e.KW != 3 || e.group_real < 0 || e.group_real > 3)) return Y5OBB_EINVAL;
    const bool grouped = e.kind >= Y5OBB_PACK_DETECT && e.kind <= Y5OBB_PACK_DETECT_BIAS;
    if (grouped && (e.group_real <= 0 || e.group_pad < e.group_real)) return Y5OBB_EINVAL;
    PackEntryK& k = h[(size_t)i];
    k.src = e.src;
    k.dst = e.dst;
    k.first = total;
    k.kind = e.kind;
    k.Cout = e.Cout;
    k.Cin = e.Cin;
    k.KH = e.KH;
    k.KW = e.KW;
    k.rows_pad = e.rows_pad;
    k.cols_pad = e.cols_pad;
    k.g_real = e.group_real;
    k.g_pad = e.group_pad;
    long long taps = (long long)e.KH * e.KW;
    if (e.kind == Y5OBB_PACK_STEM) taps = 3;
    if (e.kind == Y5OBB_PACK_DETECT_BIAS) taps = 1;
    if (e.kind == Y5OBB_PACK_DGRAD_S2) taps = ((e.group_real >> 1) ? 2 : 1) * ((e.group_real & 1) ? 2 : 1);
    total += taps * e.rows_pad * e.cols_pad;
  }
  PackPlan* p = new PackPlan();
  p->n = n;
  p->total = total;
  cudaError_t err = cudaMalloc(&p->table, sizeof(PackEntryK) * (size_t)n);
  if (err == cudaSuccess) err = cudaMemcpy(p->table, h.data(), sizeof(PackEntryK) * (size_t)n, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    if (p->table) cudaFree(p->table);
    delete p;
    return cuda_fail(err);
  }
  *out = reinterpret_cast<y5obb_pack_plan_t*>(p);
  return Y5OBB_OK;
}

int y5obb_pack_plan_run(const y5obb_pack_plan_t* plan, void* stream) {
  if (!plan) return Y5OBB_EINVAL;
  const PackPlan* p = reinterpret_cast<const PackPlan*>(plan);
  const int grid = (int)std::min<long long>((p->total + 255) / 256, (long long)sm_count() * 32);
  k_pack_weights<<<grid, 256, 0, (cudaStream_t)stream>>>(p->table, p->n, p->total);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

void y5obb_pack_plan_destroy(y5obb_pack_plan_t* plan) {
  PackPlan* p = reinterpret_cast<PackPlan*>(plan);
  if (!p) return;
  if (p->table) cudaFree(p->table);
  delete p;
}

}  // extern "C"
