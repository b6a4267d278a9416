// Weight gradient of a convolution on the tensor cores (sm_90a): for every tap (kh, kw)
//   dW[tap][co][ci] = sum over (b, ho, wo) of dz[b, ho, wo, co] * x[b, s*ho + kh - ph, s*wo + kw - pw, ci]
// i.e. a GEMM with M = Cout, N = Cin and K = all output pixels.  Both operands are read straight from the NHWC bf16
// activations / gradients (channel slices allowed): a 4-D TMA box {64 channels, kwp, khp, 1} lands in shared memory
// as [bk pixels][128 B of channels], 128B-swizzled, which is the MN-major layout wgmma reads (the reduction axis K =
// pixel rows).  The tap is a shift of the x box's origin (zero padding = TMA out-of-bounds fill, stride 2 = tensor-map
// element strides on W and H, exactly as the forward kernel reads its input).  The pixel axis is split over CTAs
// (split-K); every CTA accumulates its slice in registers (fp32) and adds it into dW with fp32 atomics.
// Replaces the cuDNN wgrad call autograd makes for the Conv layers (models/common.py) in the training step.
// Tensor-bound for wide layers (2 * pixels * Cout * Cin * taps flop), L2-bound for narrow ones.
#include <cuda.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace y5obb {
namespace {

constexpr int WG_THREADS = 384;  // two consumer warpgroups (output channels 0-63 / 64-127 of the block) + the producer warpgroup
constexpr int WG_MAX_STAGES = 8;
constexpr int WG_SMEM = 200 * 1024;
constexpr int WG_MAX_CHUNKS = 4;  // 64-column chunks of N per CTA: 4 x 64 = 256 fp32 accumulator columns per warpgroup
// a pixel block (= one TMA box per 64-channel chunk) has bk = 64 or 128 pixels; a chunk is [bk pixels][128 B]

struct WgradK {
  CUtensorMap tmA;  // dz NHWC slice: (Cout, Wo, Ho, B), box {64, kwp, khp, 1}
  CUtensorMap tmB;  // x NHWC slice: (Cin, Wi, Hi, B), box {64, kwp*s, khp*s, 1}, element strides {1, s, s, 1}
  int B, Ho, Wo, Cout, Cin;
  int KH, KW, stride, pad_h, pad_w;
  int kwp, khp, BN;         // pixel block kwp x khp = bk pixels; N tile (input channels, multiple of 16)
  int bk;                   // pixels per block (64 / 128)
  uint32_t chunk;           // bk * 128 bytes
  int tiles_w, tiles_h;     // pixel blocks per image
  int nblocks;              // B * tiles_h * tiles_w
  int T, ngroups;           // taps handled by one CTA (they share the dz tile), tap groups
  int steps;                // pipeline steps over the whole pixel axis (one pixel block each)
  int ksplit, co_blks, ci_blks;
  int stages, a_chunks, b_chunks;
  uint32_t stage_bytes;
  float* dW;                // element (tap, co, ci) at dW[tap * s_tap + row(co) * s_co + ci * s_ci]
  long long s_tap, s_co, s_ci;
  int co_group, co_group_pad;
};

// Consumer warpgroup wg: output channels cob * 128 + 64 wg + [0, 64) (A = dz chunk wg), N = the NC chunks of x (the T taps'
// tiles are consecutive 64-channel chunks: ONE N axis).  Accumulates the CTA's pixel range, then adds into dW.
template <int NC>
__device__ __forceinline__ void wgrad_consumer(const WgradK& p, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int s0,
                                               int s1, int a_chunks, int tap0, int ntap, int cob, int cib, int warp, int lane) {
  constexpr int NI = NC * 64;
  const int wg = warp >> 2;
  const uint32_t a_bytes = (uint32_t)p.a_chunks * p.chunk;
  const bool active = wg < a_chunks;  // warpgroup-uniform: this block has output channels for it
  const uint32_t ring = ptx::smem_u32(smem);
  const uint64_t desc_hi = ptx::make_mnmajor_desc(0u, p.chunk);
  const int nk = p.bk >> 4;
  float acc[NI / 2];
#pragma unroll
  for (int i = 0; i < NI / 2; ++i) acc[i] = 0.0f;
  uint32_t scale_d = 0u;
  int s = 0, prev_s = -1;
  uint32_t ph = 0;
  for (int st = s0; st < s1; ++st) {
    ptx::mbar_wait(&full_bar[s], ph);
    if (active) {
      const uint32_t sa = ring + (uint32_t)s * p.stage_bytes;
      const uint64_t da = desc_hi | (uint64_t)(((sa + (uint32_t)wg * p.chunk) & 0x3FFFFu) >> 4);
      const uint64_t db = desc_hi | (uint64_t)(((sa + a_bytes) & 0x3FFFFu) >> 4);
      ptx::wgmma_fence_regs(acc);
      ptx::wgmma_fence();
      for (int j = 0; j < nk; ++j) {  // 16 pixel rows = 2048 B per MMA
        ptx::Wgmma<NI>::template mma<1, 1>(acc, da + (uint64_t)(128 * j), db + (uint64_t)(128 * j), scale_d);
        scale_d = 1u;
      }
      ptx::wgmma_commit();
      ptx::wgmma_fence_regs(acc);
      ptx::wgmma_wait<1>();
      ptx::wgmma_fence_regs(acc);
    }
    if (prev_s >= 0) {
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty_bar[prev_s]);
    }
    prev_s = s;
    if (++s == p.stages) {
      s = 0;
      ph ^= 1u;
    }
  }
  ptx::wgmma_wait<0>();
  ptx::wgmma_fence_regs(acc);
  if (!active || s1 <= s0) return;
  // accumulator layout: thread `lane` of warp w holds rows 16 (w % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
  const int ncols = min(p.BN, p.Cin - cib * p.BN);
  const int cpt = p.b_chunks * 64;  // columns per tap
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int co = cob * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    int co_row = co;
    bool co_ok = co < p.Cout;
    if (p.co_group_pad) {
      const int a = co / p.co_group_pad, c = co - a * p.co_group_pad;
      co_ok = co_ok && c < p.co_group;
      co_row = a * p.co_group + c;
    }
    if (!co_ok) continue;
    float* row = p.dW + (long long)tap0 * p.s_tap + (long long)co_row * p.s_co + (long long)(cib * p.BN) * p.s_ci;
#pragma unroll
    for (int j = 0; j < NI / 8; ++j)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int n = 8 * j + 2 * (lane & 3) + k;
        const int t = n / cpt, ci = n - t * cpt;
        if (t < ntap && ci < ncols) atomicAdd(row + (long long)t * p.s_tap + (long long)ci * p.s_ci, acc[4 * j + 2 * i + k]);
      }
  }
}

__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_kernel(const __grid_constant__ WgradK p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[WG_MAX_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[WG_MAX_STAGES];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t WG_CHUNK = p.chunk;
  const uint32_t a_bytes = (uint32_t)p.a_chunks * WG_CHUNK, b_bytes = (uint32_t)p.b_chunks * WG_CHUNK;

  // work item: (tap group, co block, ci block, k split)
  int item = blockIdx.x;
  const int ks = item % p.ksplit;
  item /= p.ksplit;
  const int cib = item % p.ci_blks;
  item /= p.ci_blks;
  const int cob = item % p.co_blks;
  const int grp = item / p.co_blks;
  const int tap0 = grp * p.T;
  const int ntap = min(p.T, p.KH * p.KW - tap0);
  const int s0 = (int)(((long long)p.steps * ks) / p.ksplit), s1 = (int)(((long long)p.steps * (ks + 1)) / p.ksplit);
  // 64-channel chunks of A this block really has (rows of D beyond Cout are never stored)
  const int a_chunks = min(p.a_chunks, (p.Cout - cob * 128 + 63) >> 6);

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&p.tmA);
    ptx::prefetch_tmap(&p.tmB);
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
    }
    ptx::fence_mbar_init();
  }
  __syncthreads();
  const int per_img = p.tiles_h * p.tiles_w;

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 8 && ptx::elect_one()) {
      int s = 0;
      uint32_t ph = 0;
      const uint32_t tx = (uint32_t)(a_chunks + ntap * p.b_chunks) * WG_CHUNK;
      for (int st = s0; st < s1; ++st) {
        ptx::mbar_wait(&empty_bar[s], ph ^ 1u);
        uint8_t* sa = smem + (size_t)s * p.stage_bytes;
        ptx::mbar_expect_tx(&full_bar[s], tx);
        const int k = st;  // pixel block
        const int b = k / per_img;
        const int r = k - b * per_img;
        const int th = r / p.tiles_w;
        const int ho0 = th * p.khp, wo0 = (r - th * p.tiles_w) * p.kwp;
        for (int c = 0; c < a_chunks; ++c)
          ptx::tma_load_4d(sa + (size_t)c * WG_CHUNK, &p.tmA, &full_bar[s], cob * 128 + c * 64, wo0, ho0, b);
        for (int t = 0; t < ntap; ++t) {
          const int tap = tap0 + t;
          const int kh = tap / p.KW, kw = tap - kh * p.KW;
          const int wi0 = wo0 * p.stride + kw - p.pad_w, hi0 = ho0 * p.stride + kh - p.pad_h;
          uint8_t* sb = sa + a_bytes + (size_t)t * b_bytes;
          for (int c = 0; c < p.b_chunks; ++c)
            ptx::tma_load_4d(sb + (size_t)c * WG_CHUNK, &p.tmB, &full_bar[s], cib * p.BN + c * 64, wi0, hi0, b);
        }
        if (++s == p.stages) {
          s = 0;
          ph ^= 1u;
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  switch (ntap * p.b_chunks) {  // N = the chunks this CTA accumulates (the taps' x tiles are consecutive chunks)
    case 1: wgrad_consumer<1>(p, smem, full_bar, empty_bar, s0, s1, a_chunks, tap0, ntap, cob, cib, warp, lane); break;
    case 2: wgrad_consumer<2>(p, smem, full_bar, empty_bar, s0, s1, a_chunks, tap0, ntap, cob, cib, warp, lane); break;
    case 3: wgrad_consumer<3>(p, smem, full_bar, empty_bar, s0, s1, a_chunks, tap0, ntap, cob, cib, warp, lane); break;
    default: wgrad_consumer<4>(p, smem, full_bar, empty_bar, s0, s1, a_chunks, tap0, ntap, cob, cib, warp, lane); break;
  }
}

typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_tmapEncodeTiled wg_get_encode() {
  static PFN_tmapEncodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  });
  return fn;
}

struct WgradObj {
  WgradK k;
  int grid;
  size_t smem;
  double flops;
};

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_wgrad_create(const y5obb_wgrad_desc* d, y5obb_wgrad_t** out) {
  if (!d || !out || !d->dz || !d->x || !d->dw) return Y5OBB_EINVAL;
  if (d->stride != 1 && d->stride != 2) return Y5OBB_EINVAL;
  if (d->B < 1 || d->Cout < 1 || d->Cin < 1 || d->KH < 1 || d->KW < 1 || d->Ho < 1 || d->Wo < 1) return Y5OBB_EINVAL;
  if ((d->dz_pix_stride & 7) || (d->x_pix_stride & 7) || (d->x_row_stride & 7) || (d->x_img_stride & 7) ||
      d->dz_pix_stride < d->Cout)
    return Y5OBB_EINVAL;
  if ((d->x_row_stride == 0) != (d->x_img_stride == 0)) return Y5OBB_EINVAL;
  if (!d->x_row_stride && d->x_pix_stride < d->Cin) return Y5OBB_EINVAL;  // overlapping windows need explicit strides
  if ((reinterpret_cast<uintptr_t>(d->dz) | reinterpret_cast<uintptr_t>(d->x)) & 15) return Y5OBB_EINVAL;
  PFN_tmapEncodeTiled enc = wg_get_encode();
  if (!enc) return Y5OBB_ECUDA;
  WgradObj* o = new WgradObj();
  WgradK& k = o->k;
  memset(&k, 0, sizeof(k));
  k.B = d->B;
  k.Ho = d->Ho;
  k.Wo = d->Wo;
  k.Cout = d->Cout;
  k.Cin = d->Cin;
  k.KH = d->KH;
  k.KW = d->KW;
  k.stride = d->stride;
  k.pad_h = d->pad_h;
  k.pad_w = d->pad_w;
  k.dW = d->dw;
  if (d->dw_tap_stride || d->dw_co_stride || d->dw_ci_stride) {
    k.s_tap = d->dw_tap_stride;
    k.s_co = d->dw_co_stride;
    k.s_ci = d->dw_ci_stride;
  } else {
    k.s_tap = (long long)d->Cout * d->Cin;
    k.s_co = d->Cin;
    k.s_ci = 1;
  }
  if (d->co_group_pad < 0 || d->co_group < 0 || d->co_group > d->co_group_pad) {
    delete o;
    return Y5OBB_EINVAL;
  }
  k.co_group = d->co_group;
  k.co_group_pad = d->co_group_pad;
  k.ci_blks = (d->Cin + 255) / 256;
  k.BN = ((d->Cin + k.ci_blks - 1) / k.ci_blks + 15) / 16 * 16;
  k.b_chunks = (k.BN + 63) / 64;
  k.co_blks = (d->Cout + 127) / 128;
  k.a_chunks = d->Cout > 64 ? 2 : 1;
  const int ntaps = d->KH * d->KW;
  // Block size bk (pixels per TMA box) and taps per CTA T: 128-pixel blocks (fewer, larger TMA boxes), as many taps per CTA
  // as fit two pipeline stages and the WG_MAX_CHUNKS accumulator chunks (the taps share one dz tile).
  const long long npx = (long long)d->B * d->Ho * d->Wo;
  int best_bk = npx >= 512 ? 128 : 64;
  int best_T = std::max(1, std::min(ntaps, WG_MAX_CHUNKS / k.b_chunks));
  while (best_T > 1 && (uint32_t)(k.a_chunks + best_T * k.b_chunks) * (uint32_t)best_bk * 128 > WG_SMEM / 2) --best_T;
  if ((uint32_t)(k.a_chunks + best_T * k.b_chunks) * (uint32_t)best_bk * 128 > WG_SMEM / 2) best_bk = 64;
  k.bk = best_bk;
  k.chunk = (uint32_t)best_bk * 128;
  // pixel block kwp x khp = bk output pixels: the shape that covers the map with the fewest blocks (ties: widest rows)
  long long best = -1;
  for (int kwp = 1; kwp <= std::min(k.bk, 256); kwp <<= 1) {
    const int khp = k.bk / kwp;
    if (khp * d->stride > 256 || kwp * d->stride > 256) continue;  // TMA box extents (input pixels) are at most 256
    const long long cost = (long long)((d->Wo + kwp - 1) / kwp) * ((d->Ho + khp - 1) / khp);
    if (best < 0 || cost <= best) {
      best = cost;
      k.kwp = kwp;
      k.khp = khp;
    }
  }
  k.tiles_w = (d->Wo + k.kwp - 1) / k.kwp;
  k.tiles_h = (d->Ho + k.khp - 1) / k.khp;
  k.nblocks = d->B * k.tiles_w * k.tiles_h;
  const uint32_t a_bytes = (uint32_t)k.a_chunks * k.chunk, b_bytes = (uint32_t)k.b_chunks * k.chunk;
  k.ngroups = (ntaps + best_T - 1) / best_T;
  k.T = (ntaps + k.ngroups - 1) / k.ngroups;  // balanced groups
  const uint32_t blk_bytes = a_bytes + (uint32_t)k.T * b_bytes;
  if (blk_bytes > WG_SMEM / 2) {
    delete o;
    return Y5OBB_EINVAL;
  }
  k.stage_bytes = blk_bytes;
  k.stages = (int)std::min<size_t>(WG_MAX_STAGES, WG_SMEM / k.stage_bytes);
  k.steps = k.nblocks;
  const int items = k.ngroups * k.co_blks * k.ci_blks;
  {  // split-K: minimise (waves) x (steps per CTA + the fixed cost of a CTA: pipeline fill, fp32 atomic epilogue - about
     // 512 pixels' worth of pipeline steps); 1 CTA per SM
    const int sms = sm_count();  // CTAs in flight
    const int fixed = std::max(1, 512 / k.bk);
    long long best_cost2 = -1;
    int bestk = 1;
    for (int ksp = 1; ksp <= std::min(k.steps, 4 * sms); ++ksp) {
      const long long waves = ((long long)items * ksp + sms - 1) / sms;
      const long long cost = waves * ((k.steps + ksp - 1) / ksp + fixed);
      if (best_cost2 < 0 || cost < best_cost2) {
        best_cost2 = cost;
        bestk = ksp;
      }
    }
    k.ksplit = bestk;
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)d->Cout, (cuuint64_t)d->Wo, (cuuint64_t)d->Ho, (cuuint64_t)d->B};
    cuuint64_t strides[3] = {(cuuint64_t)d->dz_pix_stride * 2, (cuuint64_t)d->dz_pix_stride * d->Wo * 2,
                             (cuuint64_t)d->dz_pix_stride * d->Wo * d->Ho * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)k.kwp, (cuuint32_t)k.khp, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&k.tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->dz), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      g_last_cuda_error = (int)r;
      delete o;
      return Y5OBB_ECUDA;
    }
  }
  {
    const cuuint32_t s = (cuuint32_t)d->stride;
    cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->Wi, (cuuint64_t)d->Hi, (cuuint64_t)d->B};
    const cuuint64_t row = d->x_row_stride ? (cuuint64_t)d->x_row_stride : (cuuint64_t)d->x_pix_stride * d->Wi;
    const cuuint64_t img = d->x_img_stride ? (cuuint64_t)d->x_img_stride : row * d->Hi;
    cuuint64_t strides[3] = {(cuuint64_t)d->x_pix_stride * 2, row * 2, img * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)k.kwp * s, (cuuint32_t)k.khp * s, 1};
    cuuint32_t es[4] = {1, s, s, 1};
    CUresult r = enc(&k.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->x), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      g_last_cuda_error = (int)r;
      delete o;
      return Y5OBB_ECUDA;
    }
  }
  o->grid = items * k.ksplit;
  o->smem = (size_t)k.stages * k.stage_bytes + 1024;
  o->flops = 2.0 * d->B * d->Ho * d->Wo * (double)d->Cout * d->Cin * d->KH * d->KW;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WG_SMEM + 2048);
    if (e != cudaSuccess) {
      delete o;
      return cuda_fail(e);
    }
    attr_set = true;
  }
  *out = reinterpret_cast<y5obb_wgrad_t*>(o);
  return Y5OBB_OK;
}

int y5obb_wgrad_run(const y5obb_wgrad_t* w, void* stream) {
  if (!w) return Y5OBB_EINVAL;
  const WgradObj* o = reinterpret_cast<const WgradObj*>(w);
  wgrad_kernel<<<o->grid, WG_THREADS, o->smem, (cudaStream_t)stream>>>(o->k);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

void y5obb_wgrad_destroy(y5obb_wgrad_t* w) { delete reinterpret_cast<WgradObj*>(w); }

}  // extern "C"
