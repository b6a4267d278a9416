// HBM-bound helpers around the conv stack (NHWC bf16):
//   y5obb_stem_s2d     NCHW fp32 image -> 2x2 space-to-depth NHWC bf16 [B, H/2, W/2, 16] (12 real + 4 zero
//                      channels), which turns the 6x6/s2/p2 stem conv (models/yolov5*.yaml layer 0,
//                      models/common.py:37-49) into a 3x3/s1/p1 conv with K = 9 x 16 that the wgmma
//                      kernel runs with 32-byte swizzled tiles.
//   y5obb_sppf_pool    the three chained 5x5/s1/p2 max-pools of SPPF (models/common.py:181-196) in one
//                      pass: y1 = 5x5, y2 = 9x9, y3 = 13x13 windows of x (max-pool composition), written
//                      at channel offsets C, 2C, 3C of the same buffer (the torch.cat disappears).
//   y5obb_scale_img_s2d  scale_img (bilinear resample, optional lr flip, pad) of a test-time-augmentation branch into
//                      the same stem layout.
// Each has an fp16 form (the *_f16 entry points) for the fp16 inference plans: the stem input is then the reference's half
// image - `.half()` of an fp32 image, fp16(u * (1 / 255)) of a uint8 one (val.py:187-188: `im.half()`, then ATen's half
// `/= 255`, a multiply by the fp32 reciprocal) - and the pooled maxima are fp16 (exact either way).
// Algorithmic bytes: stem_s2d reads 12*H*W fp32 and writes H*W/4 * 32 B per image; scale_img_s2d reads the input once
// (3*H*W elements) and writes Hp*Wp/4 * 32 B per image; sppf_pool reads H*W*C*2 and writes 3x that.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "stage.cuh"

namespace y5obb {
namespace {

template <typename E>
__global__ void k_stem_s2d(const float* __restrict__ x, E* __restrict__ out, int B, int H, int W,
                           int pad_cols) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long r = i / Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    float v[16];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* p = x + (((long long)b * 3 + c) * H + 2 * ho) * W + 2 * wo;
      const float2 top = *reinterpret_cast<const float2*>(p);
      const float2 bot = *reinterpret_cast<const float2*>(p + W);
      v[0 * 3 + c] = top.x;  // (dy=0, dx=0)
      v[1 * 3 + c] = top.y;  // (dy=0, dx=1)
      v[2 * 3 + c] = bot.x;  // (dy=1, dx=0)
      v[3 * 3 + c] = bot.y;  // (dy=1, dx=1)
    }
    v[12] = v[13] = v[14] = v[15] = 0.f;
    uint4 o[2];
    pack16(v, out, o);
    // destination rows carry pad_cols zero pixels on each side (written once at allocation, never here)
    uint4* dst = reinterpret_cast<uint4*>(out + ((r * (Wo + 2 * pad_cols)) + wo + pad_cols) * 16);
    dst[0] = o[0];
    dst[1] = o[1];
  }
}

// uint8 NCHW image: the caller-side `imgs.float() / 255` (train.py:299, val.py:187-188, detect.py:108-109)
// folded into the same pass
template <typename E>
__global__ void k_stem_s2d_u8(const uint8_t* __restrict__ x, E* __restrict__ out, int B, int H, int W,
                              int pad_cols) {
  const int Ho = H >> 1, Wo = W >> 1;
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long r = i / Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    float v[16];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const uint8_t* p = x + (((long long)b * 3 + c) * H + 2 * ho) * W + 2 * wo;
      const uchar2 top = *reinterpret_cast<const uchar2*>(p);
      const uchar2 bot = *reinterpret_cast<const uchar2*>(p + W);
      v[0 * 3 + c] = u8_value(top.x, out);
      v[1 * 3 + c] = u8_value(top.y, out);
      v[2 * 3 + c] = u8_value(bot.x, out);
      v[3 * 3 + c] = u8_value(bot.y, out);
    }
    v[12] = v[13] = v[14] = v[15] = 0.f;
    uint4 o[2];
    pack16(v, out, o);
    // destination rows carry pad_cols zero pixels on each side (written once at allocation, never here)
    uint4* dst = reinterpret_cast<uint4*>(out + ((r * (Wo + 2 * pad_cols)) + wo + pad_cols) * 16);
    dst[0] = o[0];
    dst[1] = o[1];
  }
}

// scale_img (utils/torch_utils.py:239-249) of a test-time-augmentation branch, written as the stem input.  Each output pixel
// is ATen's upsample_bilinear2d_out_frame<float, float> sample (align_corners=False), with the products its sm_90 build fuses
// written as explicit _rn intrinsics so that the result does not depend on this build's contraction choices:
//   src = max(fma(scale, dst + 0.5, -0.5), 0), i0 = (int)src, i1 = i0 + (i0 < in - 1), l1 = src - i0, l0 = 1 - l1,
//   val = fma(h0l, fma(w0l, x00, w1l * x01), h1l * fma(w0l, x10, w1l * x11))
// (the second product of each sum is the plain multiply: FMUL + FFMA pairs in the sm_90 SASS torch ships).
// Pixels at or beyond (h, w) hold F.pad's value.  The left-right flip reads column W - 1 - xs of x.
__device__ __forceinline__ float ld_px(const float* p, long long i, __nv_bfloat16*) { return p[i]; }
__device__ __forceinline__ float ld_px(const uint8_t* p, long long i, __nv_bfloat16* e) { return u8_value(p[i], e); }
// fp16 plans: scale_img of the half image (upsample_bilinear2d_out_frame<Half, float>: fp16 inputs, fp32 arithmetic, one
// rounding to fp16 at the store)
__device__ __forceinline__ float ld_px(const float* p, long long i, __half*) { return __half2float(__float2half_rn(p[i])); }
__device__ __forceinline__ float ld_px(const uint8_t* p, long long i, __half* e) { return u8_value(p[i], e); }

__device__ __forceinline__ void bil_src(float scale, int dst, int in, int& i0, int& i1, float& l0, float& l1) {
  float s = __fmaf_rn(scale, (float)dst + 0.5f, -0.5f);
  s = s < 0.0f ? 0.0f : s;
  i0 = (int)s;
  i1 = i0 + (i0 < in - 1 ? 1 : 0);
  l1 = __fsub_rn(s, (float)i0);
  l0 = __fsub_rn(1.0f, l1);
}

template <typename T, typename E>
__global__ void k_scale_img_s2d(const T* __restrict__ x, E* __restrict__ out, int B, int H, int W, int h, int w,
                                int Hp, int Wp, int flip, float pad_value, float rh, float rw, int pad_cols) {
  const int Ho = Hp >> 1, Wo = Wp >> 1;
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long r = i / Wo;
    const int ho = (int)(r % Ho);
    const int b = (int)(r / Ho);
    float v[16];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const int oy = 2 * ho + dy;
      int y0, y1;
      float hl0, hl1;
      bil_src(rh, oy, H, y0, y1, hl0, hl1);
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const int ox = 2 * wo + dx;
        float* d = v + (dy * 2 + dx) * 3;
        if (oy >= h || ox >= w) {
          d[0] = d[1] = d[2] = pad_value;
          continue;
        }
        int x0, x1;
        float wl0, wl1;
        bil_src(rw, ox, W, x0, x1, wl0, wl1);
        if (flip) {  // x.flip(3)[..., xs] = x[..., W - 1 - xs]
          x0 = W - 1 - x0;
          x1 = W - 1 - x1;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const T* p = x + ((long long)b * 3 + c) * H * W;
          const long long r0 = (long long)y0 * W, r1 = (long long)y1 * W;
          const float a = __fmaf_rn(wl0, ld_px(p, r0 + x0, out), __fmul_rn(wl1, ld_px(p, r0 + x1, out)));
          const float e = __fmaf_rn(wl0, ld_px(p, r1 + x0, out), __fmul_rn(wl1, ld_px(p, r1 + x1, out)));
          d[c] = __fmaf_rn(hl0, a, __fmul_rn(hl1, e));
        }
      }
    }
    v[12] = v[13] = v[14] = v[15] = 0.f;
    uint4 o[2];
    pack16(v, out, o);
    uint4* dst = reinterpret_cast<uint4*>(out + ((r * (Wo + 2 * pad_cols)) + wo + pad_cols) * 16);
    dst[0] = o[0];
    dst[1] = o[1];
  }
}

template <typename T, typename E>
int scale_img_s2d(const T* x, void* out, int B, int H, int W, int h, int w, int Hp, int Wp, int flip, float pad_value,
                  int pad_cols, void* stream) {
  if (!x || !out || B <= 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0 || Hp <= 0 || Wp <= 0 || (Hp & 1) || (Wp & 1) ||
      h > Hp || w > Wp || pad_cols < 0)
    return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(x) & (sizeof(T) - 1)) || (reinterpret_cast<uintptr_t>(out) & 15)) return Y5OBB_EINVAL;
  // area_pixel_compute_scale (align_corners=False, no scale factor): (float)in / out, on the host as ATen does it
  const float rh = (float)H / (float)h, rw = (float)W / (float)w;
  const long long total = (long long)B * (Hp / 2) * (Wp / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_scale_img_s2d<T, E><<<grid, 256, 0, (cudaStream_t)stream>>>(x, static_cast<E*>(out), B, H, W, h, w, Hp, Wp,
                                                                flip ? 1 : 0, pad_value, rh, rw, pad_cols);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

template <typename E2>
__device__ __forceinline__ void vmax8(uint4& a, const uint4& b) {
  E2* x = reinterpret_cast<E2*>(&a);
  const E2* y = reinterpret_cast<const E2*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = __hmax2(x[i], y[i]);
}
template <typename E> struct Pair;
template <> struct Pair<__nv_bfloat16> { using T = __nv_bfloat162; static constexpr uint32_t NINF = 0xFF80FF80u; };
template <> struct Pair<__half> { using T = __half2; static constexpr uint32_t NINF = 0xFC00FC00u; };

// One CTA = one image x 8 channels x one 32x32 spatial tile (+6 halo).  Separable: a horizontal pass builds the
// 5/9/13-wide row maxima in shared memory, a vertical pass the 5/9/13-tall column maxima of those (max-pool pads
// with -inf, so clipped windows are exact).  13 + 27 shared-memory reads per pixel instead of 169 global ones.
constexpr int PT = 32, PH = 6, PIN = PT + 2 * PH;
template <typename E>
__global__ void __launch_bounds__(256) k_sppf_pool(E* __restrict__ buf, long long pix_stride, int B, int H,
                                                    int W, int C, int tiles_w, int tiles_h) {
  extern __shared__ __align__(16) uint4 sm[];
  uint4* in = sm;                       // [PIN][PIN]
  uint4* r5 = in + PIN * PIN;           // [PIN][PT]
  uint4* r9 = r5 + PIN * PT;
  uint4* r13 = r9 + PIN * PT;
  const int vec = C >> 3;
  int bid = blockIdx.x;
  const int cv = bid % vec;
  bid /= vec;
  const int tw = bid % tiles_w;
  bid /= tiles_w;
  const int th = bid % tiles_h;
  const int b = bid / tiles_h;
  const int h0 = th * PT, w0 = tw * PT;
  constexpr uint32_t NI2 = Pair<E>::NINF;
  const uint4 ninf = make_uint4(NI2, NI2, NI2, NI2);
  const E* base = buf + (long long)b * H * W * pix_stride + cv * 8;
  for (int i = threadIdx.x; i < PIN * PIN; i += 256) {
    const int y = i / PIN, x = i - y * PIN;
    const int hh = h0 + y - PH, ww = w0 + x - PH;
    uint4 v = ninf;
    if (hh >= 0 && hh < H && ww >= 0 && ww < W) v = *reinterpret_cast<const uint4*>(base + ((long long)hh * W + ww) * pix_stride);
    in[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PIN * PT; i += 256) {
    const int y = i / PT, x = i - y * PT;
    const uint4* row = in + y * PIN + x + PH;
    uint4 a5 = row[0];
    vmax8<typename Pair<E>::T>(a5, row[-1]);
    vmax8<typename Pair<E>::T>(a5, row[1]);
    vmax8<typename Pair<E>::T>(a5, row[-2]);
    vmax8<typename Pair<E>::T>(a5, row[2]);
    uint4 a9 = a5;
    vmax8<typename Pair<E>::T>(a9, row[-3]);
    vmax8<typename Pair<E>::T>(a9, row[3]);
    vmax8<typename Pair<E>::T>(a9, row[-4]);
    vmax8<typename Pair<E>::T>(a9, row[4]);
    uint4 a13 = a9;
    vmax8<typename Pair<E>::T>(a13, row[-5]);
    vmax8<typename Pair<E>::T>(a13, row[5]);
    vmax8<typename Pair<E>::T>(a13, row[-6]);
    vmax8<typename Pair<E>::T>(a13, row[6]);
    r5[i] = a5;
    r9[i] = a9;
    r13[i] = a13;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PT * PT; i += 256) {
    const int y = i / PT, x = i - y * PT;
    const int hh = h0 + y, ww = w0 + x;
    if (hh >= H || ww >= W) continue;
    const int c = (y + PH) * PT + x;
    uint4 m5 = r5[c];
    for (int d = 1; d <= 2; ++d) {
      vmax8<typename Pair<E>::T>(m5, r5[c - d * PT]);
      vmax8<typename Pair<E>::T>(m5, r5[c + d * PT]);
    }
    uint4 m9 = r9[c];
    for (int d = 1; d <= 4; ++d) {
      vmax8<typename Pair<E>::T>(m9, r9[c - d * PT]);
      vmax8<typename Pair<E>::T>(m9, r9[c + d * PT]);
    }
    uint4 m13 = r13[c];
    for (int d = 1; d <= 6; ++d) {
      vmax8<typename Pair<E>::T>(m13, r13[c - d * PT]);
      vmax8<typename Pair<E>::T>(m13, r13[c + d * PT]);
    }
    E* o = buf + (((long long)b * H + hh) * W + ww) * pix_stride + cv * 8;
    *reinterpret_cast<uint4*>(o + C) = m5;
    *reinterpret_cast<uint4*>(o + 2 * C) = m9;
    *reinterpret_cast<uint4*>(o + 3 * C) = m13;
  }
}

template <typename E>
int stem_s2d(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  if (!x_nchw || !out_nhwc16 || B <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || pad_cols < 0) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(x_nchw) & 7) || (reinterpret_cast<uintptr_t>(out_nhwc16) & 15)) return Y5OBB_EINVAL;
  const long long total = (long long)B * (H / 2) * (W / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_stem_s2d<E><<<grid, 256, 0, (cudaStream_t)stream>>>(x_nchw, static_cast<E*>(out_nhwc16), B, H, W, pad_cols);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

template <typename E>
int stem_s2d_u8(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  if (!x_nchw || !out_nhwc16 || B <= 0 || H <= 0 || W <= 0 || (H & 1) || (W & 1) || pad_cols < 0) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(x_nchw) & 1) || (reinterpret_cast<uintptr_t>(out_nhwc16) & 15)) return Y5OBB_EINVAL;
  const long long total = (long long)B * (H / 2) * (W / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_stem_s2d_u8<E><<<grid, 256, 0, (cudaStream_t)stream>>>(x_nchw, static_cast<E*>(out_nhwc16), B, H, W, pad_cols);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

template <typename E>
int sppf_pool(void* buf, int64_t pix_stride, int B, int H, int W, int C, void* stream) {
  if (!buf || B <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 7) || (pix_stride & 7) || pix_stride < 4 * (int64_t)C)
    return Y5OBB_EINVAL;
  if (reinterpret_cast<uintptr_t>(buf) & 15) return Y5OBB_EINVAL;
  const int tiles_w = (W + PT - 1) / PT, tiles_h = (H + PT - 1) / PT;
  const long long grid = (long long)B * (C / 8) * tiles_w * tiles_h;
  if (grid > 0x7FFFFFFFll) return Y5OBB_EINVAL;
  const size_t smem = (size_t)(PIN * PIN + 3 * PIN * PT) * sizeof(uint4);
  static bool attr_set = false;
  if (!attr_set) {
    Y5_CUDA(cudaFuncSetAttribute(k_sppf_pool<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_set = true;
  }
  k_sppf_pool<E><<<(unsigned)grid, 256, smem, (cudaStream_t)stream>>>(static_cast<E*>(buf), pix_stride, B, H, W, C, tiles_w,
                                                                     tiles_h);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_stem_s2d(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  return stem_s2d<__nv_bfloat16>(x_nchw, out_nhwc16, B, H, W, pad_cols, stream);
}

int y5obb_stem_s2d_u8(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  return stem_s2d_u8<__nv_bfloat16>(x_nchw, out_nhwc16, B, H, W, pad_cols, stream);
}

int y5obb_stem_s2d_f16(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  return stem_s2d<__half>(x_nchw, out_nhwc16, B, H, W, pad_cols, stream);
}

int y5obb_stem_s2d_u8_f16(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream) {
  return stem_s2d_u8<__half>(x_nchw, out_nhwc16, B, H, W, pad_cols, stream);
}

int y5obb_scale_img_s2d(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                        int flip_lr, float pad_value, int pad_cols, void* stream) {
  return scale_img_s2d<float, __nv_bfloat16>(x_nchw, out_nhwc16, B, H, W, h, w, Hp, Wp, flip_lr, pad_value, pad_cols, stream);
}

int y5obb_scale_img_s2d_u8(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                           int flip_lr, float pad_value, int pad_cols, void* stream) {
  return scale_img_s2d<uint8_t, __nv_bfloat16>(x_nchw, out_nhwc16, B, H, W, h, w, Hp, Wp, flip_lr, pad_value, pad_cols,
                                               stream);
}

int y5obb_scale_img_s2d_f16(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                            int flip_lr, float pad_value, int pad_cols, void* stream) {
  return scale_img_s2d<float, __half>(x_nchw, out_nhwc16, B, H, W, h, w, Hp, Wp, flip_lr, pad_value, pad_cols, stream);
}

int y5obb_scale_img_s2d_u8_f16(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                               int flip_lr, float pad_value, int pad_cols, void* stream) {
  return scale_img_s2d<uint8_t, __half>(x_nchw, out_nhwc16, B, H, W, h, w, Hp, Wp, flip_lr, pad_value, pad_cols, stream);
}

int y5obb_sppf_pool(void* buf, int64_t pix_stride, int B, int H, int W, int C, void* stream) {
  return sppf_pool<__nv_bfloat16>(buf, pix_stride, B, H, W, C, stream);
}

int y5obb_sppf_pool_f16(void* buf, int64_t pix_stride, int B, int H, int W, int C, void* stream) {
  return sppf_pool<__half>(buf, pix_stride, B, H, W, C, stream);
}

}  // extern "C"
