// Source images of any size -> the stem input of a batch, in one launch (the host front end of detect.py / val.py):
//   y5obb_letterbox_s2d_u8  utils/datasets.py:217-229 LoadImages.__next__ and :585-590,662-663 LoadImagesAndLabels.__getitem__:
//                           cv2.resize (utils/augmentations.py:124 INTER_LINEAR, utils/datasets.py:717-718 INTER_AREA /
//                           INTER_LINEAR) + copyMakeBorder with 114 (utils/augmentations.py:127) + HWC BGR -> CHW RGB
//                           + the `/ 255` and 2x2 space-to-depth layout of k_stem_s2d_u8.  The letterboxed uint8 image is
//                           never materialised.
// The resampled bytes are OpenCV's, bit for bit.  Its 8-bit INTER_LINEAR is fixed point (11-bit coefficient pairs per column
// and row, an int32 horizontal pass, `>> 4`, `>> 16`, `+ 2 >> 2` in the vertical pass), so it is order-free; the coefficient
// tables are O(new_w + new_h) per image and come from the host (letterbox.py), formed in the float types OpenCV uses.
// INTER_AREA by an integer factor is an integer block sum (2x2: (sum + 2) >> 2; otherwise the fp32 product sum * (1.f / area)
// rounded half to even); by a fractional factor it is an fp32 accumulation in OpenCV's order: per source row the weighted
// columns in table order, then the weighted rows in table order, every product and sum rounded separately (no FMA).
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "stage.cuh"

namespace y5obb {
namespace {

using Desc = y5obb_letterbox_desc;

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// resized pixel (y, x) of image d -> px (BGR, as stored)
__device__ __forceinline__ void lb_pixel(const Desc& d, const uint8_t* __restrict__ src, const int32_t* __restrict__ tab, int y,
                                         int x, uint8_t px[3]) {
  const long long w0 = d.w0;
  if (d.mode == Y5OBB_LB_COPY) {
    const uint8_t* p = src + ((long long)y * w0 + x) * 3;
    px[0] = p[0], px[1] = p[1], px[2] = p[2];
  } else if (d.mode == Y5OBB_LB_LINEAR) {
    const int32_t* tx = tab + d.xtab + 2 * x;
    const int32_t* ty = tab + d.ytab + 2 * y;
    const int sx0 = clampi(tx[0], 0, d.w0 - 1), sx1 = min(sx0 + 1, d.w0 - 1);
    const int r0 = clampi(ty[0], 0, d.h0 - 1), r1 = clampi(ty[0] + 1, 0, d.h0 - 1);
    const int a0 = (short)(tx[1] & 0xffff), a1 = tx[1] >> 16, b0 = (short)(ty[1] & 0xffff), b1 = ty[1] >> 16;
    const uint8_t *p00 = src + (r0 * w0 + sx0) * 3, *p01 = src + (r0 * w0 + sx1) * 3;
    const uint8_t *p10 = src + (r1 * w0 + sx0) * 3, *p11 = src + (r1 * w0 + sx1) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = p00[c] * a0 + p01[c] * a1, h1 = p10[c] * a0 + p11[c] * a1;
      const int v = ((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16);
      px[c] = (uint8_t)clampi((v + 2) >> 2, 0, 255);
    }
  } else if (d.mode == Y5OBB_LB_AREA_INT) {
    int sum[3] = {0, 0, 0};
    const uint8_t* p = src + ((long long)y * d.ky * w0 + (long long)x * d.kx) * 3;
    for (int j = 0; j < d.ky; ++j, p += w0 * 3)
      for (int k = 0; k < d.kx; ++k) {
        sum[0] += p[3 * k], sum[1] += p[3 * k + 1], sum[2] += p[3 * k + 2];
      }
#pragma unroll
    for (int c = 0; c < 3; ++c)
      px[c] = (d.kx == 2 && d.ky == 2) ? (uint8_t)((sum[c] + 2) >> 2)
                                       : (uint8_t)clampi(__float2int_rn(__fmul_rn((float)sum[c], d.inv_area)), 0, 255);
  } else {  // Y5OBB_LB_AREA: [n + 1] first-tap indices, then (source index, fp32 weight) pairs
    const int32_t *xf = tab + d.xtab, *yf = tab + d.ytab;
    const int32_t *xe = xf + d.new_w + 1, *ye = yf + d.new_h + 1;
    const int k0 = xf[x], k1 = xf[x + 1], j0 = yf[y], j1 = yf[y + 1];
    float acc[3] = {0.f, 0.f, 0.f};
    for (int j = j0; j < j1; ++j) {
      const uint8_t* row = src + (long long)clampi(ye[2 * j], 0, d.h0 - 1) * w0 * 3;
      const float beta = __int_as_float(ye[2 * j + 1]);
      float buf[3] = {0.f, 0.f, 0.f};
      for (int k = k0; k < k1; ++k) {
        const uint8_t* p = row + clampi(xe[2 * k], 0, d.w0 - 1) * 3;
        const float alpha = __int_as_float(xe[2 * k + 1]);
#pragma unroll
        for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)p[c], alpha));
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) acc[c] = j == j0 ? __fmul_rn(beta, buf[c]) : __fadd_rn(acc[c], __fmul_rn(beta, buf[c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) px[c] = (uint8_t)clampi(__float2int_rn(acc[c]), 0, 255);
  }
}

template <typename E>
__global__ void k_letterbox_s2d_u8(const uint8_t* __restrict__ src, const Desc* __restrict__ desc, int B, int Hp, int Wp,
                                   E* __restrict__ out, int pad_cols) {
  const int Ho = Hp >> 1, Wo = Wp >> 1;
  const int32_t* tab = reinterpret_cast<const int32_t*>(desc);
  const long long total = (long long)B * Ho * Wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int wo = (int)(i % Wo);
    const long long r = i / Wo;
    const int ho = (int)(r % Ho);
    const Desc d = desc[(int)(r / Ho)];
    float v[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int y = 2 * ho + (q >> 1) - d.top, x = 2 * wo + (q & 1) - d.left;
      uint8_t px[3] = {114, 114, 114};
      if (y >= 0 && y < d.new_h && x >= 0 && x < d.new_w) lb_pixel(d, src + d.src_off, tab, y, x, px);
      v[q * 3] = u8_value(px[2], out);  // BGR -> RGB
      v[q * 3 + 1] = u8_value(px[1], out);
      v[q * 3 + 2] = u8_value(px[0], out);
    }
    v[12] = v[13] = v[14] = v[15] = 0.f;
    uint4 o[2];
    pack16(v, out, o);
    uint4* dst = reinterpret_cast<uint4*>(out + ((r * (Wo + 2 * pad_cols)) + wo + pad_cols) * 16);
    dst[0] = o[0];
    dst[1] = o[1];
  }
}

// whether the fixed part of one axis' table lies inside the buffer of `words` 32-bit words
bool table_fits(int mode, int off, int n, int64_t words) {
  if (mode == Y5OBB_LB_LINEAR) return off >= 0 && (int64_t)off + 2ll * n <= words;
  if (mode == Y5OBB_LB_AREA) return off >= 0 && (int64_t)off + n + 1 <= words;  // (its tap list is checked by the caller)
  return true;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

static int letterbox_s2d_u8(bool f16, const uint8_t* src, int64_t src_bytes, const void* desc_dev,
                            const y5obb_letterbox_desc* desc_host, int64_t desc_bytes, int B, int Hp, int Wp, void* out_nhwc16,
                            int pad_cols, void* stream) {
  if (!src || !desc_dev || !desc_host || !out_nhwc16 || B <= 0 || Hp <= 0 || Wp <= 0 || (Hp & 1) || (Wp & 1) || pad_cols < 0 ||
      src_bytes <= 0 || desc_bytes < (int64_t)B * (int64_t)sizeof(y5obb_letterbox_desc) || (desc_bytes & 3))
    return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(out_nhwc16) & 15) || (reinterpret_cast<uintptr_t>(desc_dev) & 7)) return Y5OBB_EINVAL;
  const int64_t words = desc_bytes / 4;
  for (int b = 0; b < B; ++b) {
    const y5obb_letterbox_desc& d = desc_host[b];
    if (d.h0 <= 0 || d.w0 <= 0 || d.new_h <= 0 || d.new_w <= 0 || d.top < 0 || d.left < 0 || d.top + (int64_t)d.new_h > Hp ||
        d.left + (int64_t)d.new_w > Wp || d.src_off < 0 || d.src_off + (int64_t)d.h0 * d.w0 * 3 > src_bytes)
      return Y5OBB_EINVAL;
    switch (d.mode) {
      case Y5OBB_LB_COPY:
        if (d.new_h != d.h0 || d.new_w != d.w0) return Y5OBB_EINVAL;
        break;
      case Y5OBB_LB_AREA_INT:
        if (d.kx < 1 || d.ky < 1 || (int64_t)d.new_w * d.kx > d.w0 || (int64_t)d.new_h * d.ky > d.h0) return Y5OBB_EINVAL;
        break;
      case Y5OBB_LB_AREA:
        if (d.new_w > d.w0 || d.new_h > d.h0) return Y5OBB_EINVAL;
        break;
      case Y5OBB_LB_LINEAR:
        break;
      default:
        return Y5OBB_EINVAL;
    }
    if (!table_fits(d.mode, d.xtab, d.new_w, words) || !table_fits(d.mode, d.ytab, d.new_h, words)) return Y5OBB_EINVAL;
    if (d.mode == Y5OBB_LB_AREA) {  // the tap lists: first-tap indices ascending from 0, the last one inside the buffer
      const int32_t* w32 = reinterpret_cast<const int32_t*>(desc_host);
      const int32_t *xf = w32 + d.xtab, *yf = w32 + d.ytab;
      if (xf[0] != 0 || yf[0] != 0) return Y5OBB_EINVAL;
      for (int i = 0; i < d.new_w; ++i)
        if (xf[i + 1] < xf[i]) return Y5OBB_EINVAL;
      for (int i = 0; i < d.new_h; ++i)
        if (yf[i + 1] < yf[i]) return Y5OBB_EINVAL;
      if ((int64_t)d.xtab + d.new_w + 1 + 2ll * xf[d.new_w] > words || (int64_t)d.ytab + d.new_h + 1 + 2ll * yf[d.new_h] > words)
        return Y5OBB_EINVAL;
    }
  }
  const long long total = (long long)B * (Hp / 2) * (Wp / 2);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  const Desc* dd = static_cast<const y5obb_letterbox_desc*>(desc_dev);
  if (f16)
    k_letterbox_s2d_u8<<<grid, 256, 0, (cudaStream_t)stream>>>(src, dd, B, Hp, Wp, static_cast<__half*>(out_nhwc16), pad_cols);
  else
    k_letterbox_s2d_u8<<<grid, 256, 0, (cudaStream_t)stream>>>(src, dd, B, Hp, Wp, static_cast<__nv_bfloat16*>(out_nhwc16),
                                                              pad_cols);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_letterbox_s2d_u8(const uint8_t* src, int64_t src_bytes, const void* desc_dev, const y5obb_letterbox_desc* desc_host,
                           int64_t desc_bytes, int B, int Hp, int Wp, void* out_nhwc16, int pad_cols, void* stream) {
  return letterbox_s2d_u8(false, src, src_bytes, desc_dev, desc_host, desc_bytes, B, Hp, Wp, out_nhwc16, pad_cols, stream);
}

int y5obb_letterbox_s2d_u8_f16(const uint8_t* src, int64_t src_bytes, const void* desc_dev, const y5obb_letterbox_desc* desc_host,
                               int64_t desc_bytes, int B, int Hp, int Wp, void* out_nhwc16, int pad_cols, void* stream) {
  return letterbox_s2d_u8(true, src, src_bytes, desc_dev, desc_host, desc_bytes, B, Hp, Wp, out_nhwc16, pad_cols, stream);
}

}  // extern "C"
