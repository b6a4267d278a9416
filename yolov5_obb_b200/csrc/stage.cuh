// Stem-input staging shared by the kernels that write the space-to-depth image (aux_kernels.cu, letterbox.cu, scene.cu):
// 16 channels rounded to the plan's element type - bf16, or fp16 for the fp16 plans (Y5OBB_CONV_F16) - and the value of a
// uint8 image sample.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace y5obb {

// 16 stem channels as two 16-byte vectors
__device__ __forceinline__ void pack16(const float (&v)[16], __nv_bfloat16*, uint4 (&o)[2]) {
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(o);
#pragma unroll
  for (int e = 0; e < 8; ++e) h[e] = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
}
__device__ __forceinline__ void pack16(const float (&v)[16], __half*, uint4 (&o)[2]) {
  __half2* h = reinterpret_cast<__half2*>(o);
#pragma unroll
  for (int e = 0; e < 8; ++e) h[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
}
// a uint8 image sample: bf16 plans divide by 255 in fp32; fp16 plans take the reference's half image, `im.half()` (exact)
// then ATen's half `/= 255`, which multiplies by the fp32 reciprocal and rounds once to fp16 (val.py:187-188)
__device__ __forceinline__ float u8_value(uint8_t u, __nv_bfloat16*) { return (float)u / 255.0f; }
__device__ __forceinline__ float u8_value(uint8_t u, __half*) {
  return __half2float(__float2half_rn(__fmul_rn((float)u, 1.0f / 255.0f)));
}

}  // namespace y5obb
