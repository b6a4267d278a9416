// Shared host/device helpers for liby5obb (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/y5obb.h"

namespace y5obb {

extern thread_local int g_last_cuda_error;

inline int cuda_fail(cudaError_t e) {
  g_last_cuda_error = (int)e;
  return Y5OBB_ECUDA;
}

#define Y5_CUDA(expr)                                   \
  do {                                                  \
    cudaError_t _e = (expr);                            \
    if (_e != cudaSuccess) return ::y5obb::cuda_fail(_e); \
  } while (0)

#define Y5_LAUNCH_CHECK() Y5_CUDA(cudaGetLastError())

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator over a caller-provided workspace.
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base(static_cast<char*>(p)) {}
  template <typename T>
  T* take(size_t count) {
    off = align_up(off, 256);
    T* p = reinterpret_cast<T*>(base + off);
    off += count * sizeof(T);
    return p;
  }
  size_t used() const { return align_up(off, 256); }
};

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace y5obb
