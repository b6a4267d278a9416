// Training-mode BatchNorm + SiLU around the tensor-core convolution (NHWC bf16), forward and backward.
// Replaces the cuDNN/ATen batch_norm + SiLU kernels behind models/common.py:45-46
// (Conv.forward = act(bn(conv(x)))) in train mode (train.py:324-333), with BN eps = 1e-3 and momentum = 0.03
// (utils/torch_utils.py:160-162).
//
// forward:   z = conv(x) (tensor-core kernel, raw bf16)                     [conv_sm90.cu]
//            k_bn_stats      per-channel sum / sum of squares of z (fp32 atomics, one pass over z)
//            k_bn_finalize   mean, biased var -> scale = gamma / sqrt(var + eps), shift = beta - mean * scale;
//                            running_mean / running_var update (unbiased var), as torch.nn.BatchNorm2d
//            k_bn_silu_apply y = [res +] silu(z * scale + shift) written to a channel slice (+ optional 2x up-sampled copy)
// backward:  k_bn_silu_bwd_reduce   dz_hat = dy * silu'(u), u = z*scale+shift; per-channel sum(dz_hat), sum(dz_hat * xhat)
//            k_bn_silu_bwd_apply    dz = scale * (dz_hat - mean(dz_hat) - xhat * mean(dz_hat * xhat)); dgamma, dbeta
// All HBM-bound: algorithmic bytes per element are 2 (read z) for stats, 2 + 2 for apply (+2 with a residual).
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace y5obb {
namespace {

constexpr int STAT_THREADS = 256;

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return o;
}

// Per-channel reductions over the pixels of an NHWC bf16 slice, deterministic: block b reduces the contiguous pixel
// range [b * chunk, (b + 1) * chunk) and STORES its partial sums to partial[b][2][C]; k_reduce_partials then adds the
// partials in block order.  (fp32 atomics would make the statistics - and, through the chaotic amplification of a
// freshly initialised BatchNorm network, the whole step - differ from run to run.)
// Thread layout: `cols` threads side by side cover the 8-channel vectors of one pixel (coalesced 16-byte loads),
// `lanes` = 256 / cols pixels are in flight per block.
__device__ __forceinline__ void block_partials(float (&s)[8], float (&q)[8], float (*red)[STAT_THREADS][8], int cols, int lanes,
                                               int col_in, int lane, bool active_col, int cv, int C,
                                               float* __restrict__ partial) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    red[0][threadIdx.x][k] = s[k];
    red[1][threadIdx.x][k] = q[k];
  }
  __syncthreads();
  // the first 16 lanes of each column add every 16th lane, then lane 0 adds those 16 (fixed order)
  if (lane < 16 && active_col) {
    for (int l = lane + 16; l < lanes; l += 16) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s[k] += red[0][l * cols + col_in][k];
        q[k] += red[1][l * cols + col_in][k];
      }
    }
  }
  __syncthreads();
  if (lane < 16 && lane > 0 && active_col) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      red[0][threadIdx.x][k] = s[k];
      red[1][threadIdx.x][k] = q[k];
    }
  }
  __syncthreads();
  if (lane == 0 && active_col) {
    for (int l = 1; l < min(16, lanes); ++l) {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s[k] += red[0][l * cols + col_in][k];
        q[k] += red[1][l * cols + col_in][k];
      }
    }
    float* o = partial + (long long)blockIdx.x * 2 * C + cv * 8;
    *reinterpret_cast<float4*>(o) = make_float4(s[0], s[1], s[2], s[3]);
    *reinterpret_cast<float4*>(o + 4) = make_float4(s[4], s[5], s[6], s[7]);
    *reinterpret_cast<float4*>(o + C) = make_float4(q[0], q[1], q[2], q[3]);
    *reinterpret_cast<float4*>(o + C + 4) = make_float4(q[4], q[5], q[6], q[7]);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(STAT_THREADS) k_bn_stats(const __nv_bfloat16* __restrict__ z, long long pix_stride,
                                                           long long npix, int C, long long chunk,
                                                           float* __restrict__ partial) {
  const int vecs = C >> 3;
  const int cols = min(vecs, STAT_THREADS);         // vector columns handled per pass by this block
  const int lanes = STAT_THREADS / cols;            // pixel lanes per column
  const int col_in = threadIdx.x % cols, lane = threadIdx.x / cols;
  __shared__ float red[2][STAT_THREADS][8];
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  for (int cv0 = 0; cv0 < vecs; cv0 += cols) {
    const int cv = cv0 + col_in;
    const bool active = cv < vecs && lane < lanes;
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
      const __nv_bfloat16* base = z + cv * 8;
      long long p = p0 + lane;
      for (; p + 3LL * lanes < p1; p += 4LL * lanes) {  // four independent 16-byte loads in flight
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const uint4*>(base + (p + (long long)u * lanes) * pix_stride);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float f[8];
          unpack8(v[u], f);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            s[k] += f[k];
            q[k] = fmaf(f[k], f[k], q[k]);
          }
        }
      }
      for (; p < p1; p += lanes) {
        float f[8];
        unpack8(*reinterpret_cast<const uint4*>(base + p * pix_stride), f);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          s[k] += f[k];
          q[k] = fmaf(f[k], f[k], q[k]);
        }
      }
    }
    block_partials(s, q, red, cols, lanes, col_in, lane, active, cv, C, partial);
  }
}

// out[j] = sum over blocks of partial[b][j], j in [0, 2C): [0, C) -> out_a, [C, 2C) -> out_b, in a FIXED order: thread
// (seg, col) adds rows seg, seg + 32, ... and thread (0, col) then adds the 32 segment sums.  8 columns x 32 row
// segments per block.  Optionally also writes the BatchNorm parameter gradients dgamma (+)= out_b, dbeta (+)= out_a.
// T = double: the fp32 sums are widened once, into a SyncBatchNorm record (k_reduce_partials_rec).
template <typename T>
__device__ __forceinline__ void reduce_partials(const float* __restrict__ partial, int blocks, int C, T* __restrict__ out_a,
                                                T* __restrict__ out_b, float* __restrict__ dgamma,
                                                float* __restrict__ dbeta, int param_accumulate) {
  __shared__ float red[32][8];
  const int col = threadIdx.x & 7, seg = threadIdx.x >> 3;
  const int j = blockIdx.x * 8 + col;
  float acc = 0.f;
  if (j < 2 * C)
    for (int b = seg; b < blocks; b += 32) acc += partial[(long long)b * 2 * C + j];
  red[seg][col] = acc;
  __syncthreads();
  if (seg == 0 && j < 2 * C) {
    float t = red[0][col];
#pragma unroll
    for (int s2 = 1; s2 < 32; ++s2) t += red[s2][col];
    if (j < C) {
      out_a[j] = t;
      if (dbeta) dbeta[j] = (param_accumulate ? dbeta[j] : 0.f) + t;
    } else {
      out_b[j - C] = t;
      if (dgamma) dgamma[j - C] = (param_accumulate ? dgamma[j - C] : 0.f) + t;
    }
  }
}

__global__ void __launch_bounds__(256) k_reduce_partials(const float* __restrict__ partial, int blocks, int C,
                                                         float* __restrict__ out_a, float* __restrict__ out_b,
                                                         float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                         int param_accumulate) {
  reduce_partials(partial, blocks, C, out_a, out_b, dgamma, dbeta, param_accumulate);
}

// SyncBatchNorm backward, first half: the rank's record [sum(du) (C) | sum(du * xhat) (C)] in fp64, local dgamma / dbeta
__global__ void __launch_bounds__(256) k_reduce_partials_rec(const float* __restrict__ partial, int blocks, int C,
                                                             double* __restrict__ rec, float* __restrict__ dgamma,
                                                             float* __restrict__ dbeta, int param_accumulate) {
  reduce_partials(partial, blocks, C, rec, rec + C, dgamma, dbeta, param_accumulate);
}

// k_reduce_partials + k_bn_finalize in one launch: thread (seg, col) adds rows seg, seg + 32, ... of BOTH statistics of
// channel c, thread (0, col) adds the 32 segment sums in order and finalises the channel.
// RECORD (k_reduce_stats_rec): the thread stores the sums instead, as the rank's SyncBatchNorm record
// rec[2C + 1] = [sum (C) | sum of squares (C) | n] in fp64 (the fp32 sums widened once; an fp32 count would be inexact
// above 2^24 pixels), which k_bn_finalize_rec finalises once every rank's record is added in.
template <bool RECORD>
__device__ __forceinline__ void reduce_finalize(const float* __restrict__ partial, int blocks, long long npix, int C,
                                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                float momentum, float* __restrict__ running_mean,
                                                float* __restrict__ running_var, float* __restrict__ scale,
                                                float* __restrict__ shift, float* __restrict__ mean_out,
                                                float* __restrict__ invstd_out, double* __restrict__ rec) {
  __shared__ float red[2][32][8];
  const int col = threadIdx.x & 7, seg = threadIdx.x >> 3;
  const int c = blockIdx.x * 8 + col;
  float a = 0.f, b = 0.f;
  if (c < C)
    for (int r = seg; r < blocks; r += 32) {
      a += partial[(long long)r * 2 * C + c];
      b += partial[(long long)r * 2 * C + C + c];
    }
  red[0][seg][col] = a;
  red[1][seg][col] = b;
  __syncthreads();
  if (seg != 0 || c >= C) return;
  float sum = red[0][0][col], sumsq = red[1][0][col];
#pragma unroll
  for (int s2 = 1; s2 < 32; ++s2) {
    sum += red[0][s2][col];
    sumsq += red[1][s2][col];
  }
  if (RECORD) {
    rec[c] = (double)sum;
    rec[C + c] = (double)sumsq;
    if (c == 0) rec[2 * C] = (double)npix;
    return;
  }
  const double n = (double)npix;
  const double m = (double)sum / n;
  double var = (double)sumsq / n - m * m;
  if (var < 0) var = 0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - (float)m * sc;
  mean_out[c] = (float)m;
  invstd_out[c] = invstd;
  if (running_mean) {
    const double unbiased = n > 1 ? var * n / (n - 1.0) : var;
    running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * (float)m;
    running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

__global__ void __launch_bounds__(256) k_reduce_finalize(const float* __restrict__ partial, int blocks, long long npix, int C,
                                                         const float* __restrict__ gamma, const float* __restrict__ beta,
                                                         float eps, float momentum, float* __restrict__ running_mean,
                                                         float* __restrict__ running_var, float* __restrict__ scale,
                                                         float* __restrict__ shift, float* __restrict__ mean_out,
                                                         float* __restrict__ invstd_out) {
  reduce_finalize<false>(partial, blocks, npix, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift,
                         mean_out, invstd_out, nullptr);
}

__global__ void __launch_bounds__(256) k_reduce_stats_rec(const float* __restrict__ partial, int blocks, long long npix, int C,
                                                          double* __restrict__ rec) {
  reduce_finalize<true>(partial, blocks, npix, C, nullptr, nullptr, 0.f, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr,
                        nullptr, rec);
}

// mean, biased var -> invstd, scale, shift; running statistics with the unbiased var over n pixels (torch.nn.BatchNorm2d).
// S = double (k_bn_finalize_rec): sums and count from a SyncBatchNorm record added over every rank.
template <typename S>
__device__ __forceinline__ void bn_finalize(const S* __restrict__ sum, const S* __restrict__ sumsq, long long npix,
                                            const double* __restrict__ n_all, int C, const float* __restrict__ gamma,
                                            const float* __restrict__ beta, float eps, float momentum,
                                            float* __restrict__ running_mean, float* __restrict__ running_var,
                                            float* __restrict__ scale, float* __restrict__ shift,
                                            float* __restrict__ mean_out, float* __restrict__ invstd_out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double n;
  if constexpr (std::is_same<S, double>::value)
    n = *n_all;
  else
    n = (double)npix;
  const double m = (double)sum[c] / n;
  double var = (double)sumsq[c] / n - m * m;
  if (var < 0) var = 0;
  const float invstd = (float)(1.0 / sqrt(var + (double)eps));
  const float sc = gamma[c] * invstd;
  scale[c] = sc;
  shift[c] = beta[c] - (float)m * sc;
  mean_out[c] = (float)m;
  invstd_out[c] = invstd;
  if (running_mean) {
    const double unbiased = n > 1 ? var * n / (n - 1.0) : var;
    running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * (float)m;
    running_var[c] = (1.0f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}

__global__ void k_bn_finalize(const float* __restrict__ sum, const float* __restrict__ sumsq, long long npix, int C,
                              const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                              float* __restrict__ running_mean, float* __restrict__ running_var,
                              float* __restrict__ scale, float* __restrict__ shift, float* __restrict__ mean_out,
                              float* __restrict__ invstd_out) {
  bn_finalize(sum, sumsq, npix, nullptr, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift, mean_out,
              invstd_out);
}

// SyncBatchNorm forward, second half: rec = the records of every rank added up (its sums and its count rec[2C])
__global__ void k_bn_finalize_rec(const double* __restrict__ rec, int C, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, float eps, float momentum, float* __restrict__ running_mean,
                                  float* __restrict__ running_var, float* __restrict__ scale, float* __restrict__ shift,
                                  float* __restrict__ mean_out, float* __restrict__ invstd_out) {
  bn_finalize(rec, rec + C, 0, rec + 2 * C, C, gamma, beta, eps, momentum, running_mean, running_var, scale, shift, mean_out,
              invstd_out);
}

// sigmoid through the hardware tanh (one MUFU op, |rel err| ~ 2^-11: far below the bf16 the results are stored in)
__device__ __forceinline__ float sigmoid_tanh(float u) {
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(0.5f * u));
  return fmaf(0.5f, t, 0.5f);
}
__device__ __forceinline__ float silu_f(float u) { return u * sigmoid_tanh(u); }

// Column-persistent element-wise kernels: a thread keeps ONE 8-channel vector column (its per-channel coefficients live
// in registers) and walks over pixels; `cols` threads side by side cover a pixel's vectors (coalesced), 256 / cols pixels
// per block step.  blockIdx.y selects the group of `cols` columns when C / 8 > 256.
__global__ void __launch_bounds__(256) k_bn_silu_apply(const __nv_bfloat16* __restrict__ z, long long z_stride, long long npix,
                                                       int C, int W, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, int act,
                                                       const __nv_bfloat16* __restrict__ res, long long res_stride,
                                                       __nv_bfloat16* __restrict__ y, long long y_stride,
                                                       __nv_bfloat16* __restrict__ y2x, long long y2x_stride) {
  const int vecs = C >> 3;
  const int cols = min(vecs, 256);
  const int lanes = 256 / cols;
  const int col_in = threadIdx.x % cols, lane = threadIdx.x / cols;
  const int cv = blockIdx.y * cols + col_in;
  if (cv >= vecs || lane >= lanes) return;
  float sc[8], sh[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    sc[k] = scale[cv * 8 + k];
    sh[k] = shift[cv * 8 + k];
  }
  const long long step = (long long)gridDim.x * lanes;
  for (long long p = (long long)blockIdx.x * lanes + lane; p < npix; p += 2 * step) {
    const long long p2 = p + step;
    const bool two = p2 < npix;
    const uint4 v0 = *reinterpret_cast<const uint4*>(z + p * z_stride + cv * 8);
    uint4 v1 = make_uint4(0, 0, 0, 0), r0 = v1, r1 = v1;
    if (two) v1 = *reinterpret_cast<const uint4*>(z + p2 * z_stride + cv * 8);
    if (res) {
      r0 = *reinterpret_cast<const uint4*>(res + p * res_stride + cv * 8);
      if (two) r1 = *reinterpret_cast<const uint4*>(res + p2 * res_stride + cv * 8);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two) break;
      const long long q = h ? p2 : p;
      float f[8];
      unpack8(h ? v1 : v0, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float u = fmaf(f[k], sc[k], sh[k]);
        f[k] = act ? silu_f(u) : u;
      }
      if (res) {
        float r[8];
        unpack8(h ? r1 : r0, r);
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] += r[k];
      }
      const uint4 o = pack8(f);
      *reinterpret_cast<uint4*>(y + q * y_stride + cv * 8) = o;
      if (y2x) {  // nearest 2x up-sampled copy: pixel (b, h, w) -> (b, 2h + {0,1}, 2w + {0,1})
        const long long row = q / W;  // b * H + h
        const int w = (int)(q - row * W);
        __nv_bfloat16* u0 = y2x + ((row * 2) * (2LL * W) + 2 * w) * y2x_stride + cv * 8;
        *reinterpret_cast<uint4*>(u0) = o;
        *reinterpret_cast<uint4*>(u0 + y2x_stride) = o;
        *reinterpret_cast<uint4*>(u0 + 2LL * W * y2x_stride) = o;
        *reinterpret_cast<uint4*>(u0 + 2LL * W * y2x_stride + y2x_stride) = o;
      }
    }
  }
}


__device__ __forceinline__ float silu_grad(float u) {
  const float sg = sigmoid_tanh(u);
  return fmaf(u * sg, 1.0f - sg, sg);
}

// per-channel sum(du) and sum(du * xhat), du = dy * act'(u), u = z*scale + shift, xhat = (z - mean) * invstd
// (block partials as k_bn_stats)
__global__ void __launch_bounds__(STAT_THREADS) k_bn_bwd_reduce(const __nv_bfloat16* __restrict__ z, long long z_stride,
                                                                const __nv_bfloat16* __restrict__ dy, long long dy_stride,
                                                                long long npix, int C, const float* __restrict__ scale,
                                                                const float* __restrict__ shift,
                                                                const float* __restrict__ mean,
                                                                const float* __restrict__ invstd, int act, long long chunk,
                                                                float* __restrict__ partial) {
  const int vecs = C >> 3;
  const int cols = min(vecs, STAT_THREADS);
  const int lanes = STAT_THREADS / cols;
  const int col_in = threadIdx.x % cols, lane = threadIdx.x / cols;
  __shared__ float red[2][STAT_THREADS][8];
  const long long p0 = (long long)blockIdx.x * chunk, p1 = min(npix, p0 + chunk);
  for (int cv0 = 0; cv0 < vecs; cv0 += cols) {
    const int cv = cv0 + col_in;
    const bool active = cv < vecs && lane < lanes;
    float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
      float sc[8], sh[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        sc[k] = scale[cv * 8 + k];
        sh[k] = shift[cv * 8 + k];
      }
      const __nv_bfloat16* zb = z + cv * 8;
      const __nv_bfloat16* db = dy + cv * 8;
      // q accumulates sum(du * z); sum(du * xhat) = invstd * (sum(du * z) - mean * sum(du)) is formed once per block
      long long p = p0 + lane;
      for (; p + lanes < p1; p += 2LL * lanes) {  // two pixels (four 16-byte loads) in flight
        const uint4 z0 = *reinterpret_cast<const uint4*>(zb + p * z_stride);
        const uint4 d0 = *reinterpret_cast<const uint4*>(db + p * dy_stride);
        const uint4 z1 = *reinterpret_cast<const uint4*>(zb + (p + lanes) * z_stride);
        const uint4 d1 = *reinterpret_cast<const uint4*>(db + (p + lanes) * dy_stride);
        float zf[8], df[8];
        unpack8(z0, zf);
        unpack8(d0, df);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float du = act ? df[k] * silu_grad(fmaf(zf[k], sc[k], sh[k])) : df[k];
          s[k] += du;
          q[k] = fmaf(du, zf[k], q[k]);
        }
        unpack8(z1, zf);
        unpack8(d1, df);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float du = act ? df[k] * silu_grad(fmaf(zf[k], sc[k], sh[k])) : df[k];
          s[k] += du;
          q[k] = fmaf(du, zf[k], q[k]);
        }
      }
      for (; p < p1; p += lanes) {
        float zf[8], df[8];
        unpack8(*reinterpret_cast<const uint4*>(zb + p * z_stride), zf);
        unpack8(*reinterpret_cast<const uint4*>(db + p * dy_stride), df);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float du = act ? df[k] * silu_grad(fmaf(zf[k], sc[k], sh[k])) : df[k];
          s[k] += du;
          q[k] = fmaf(du, zf[k], q[k]);
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) q[k] = invstd[cv * 8 + k] * (q[k] - mean[cv * 8 + k] * s[k]);
    }
    block_partials(s, q, red, cols, lanes, col_in, lane, active, cv, C, partial);
  }
}

// dz = scale * (du - sum_du / N - xhat * sum_dux / N) = k1 * du + k2 * z + k3 with per-channel k1 = scale,
// k2 = -scale * invstd * sum_dux / N, k3 = scale * (mean * invstd * sum_dux / N - sum_du / N);
// optional pass-through of dy into the residual branch.  Column-persistent threads (see k_bn_silu_apply).
// S = double (k_bn_bwd_apply_rec): the sums come from a SyncBatchNorm record summed over every rank and N is the forward
// record's count `n_all`; the loop still covers the npix local pixels.
template <typename S>
__device__ __forceinline__ void bn_bwd_apply(const __nv_bfloat16* __restrict__ z, long long z_stride,
                                             const __nv_bfloat16* __restrict__ dy, long long dy_stride, long long npix, int C,
                                             const float* __restrict__ scale, const float* __restrict__ shift,
                                             const float* __restrict__ mean, const float* __restrict__ invstd, int act,
                                             const S* __restrict__ sum_du, const S* __restrict__ sum_dux,
                                             const double* __restrict__ n_all, __nv_bfloat16* __restrict__ dz,
                                             long long dz_stride, __nv_bfloat16* __restrict__ gres, long long gres_stride,
                                             int gres_accumulate) {
  const int vecs = C >> 3;
  const int cols = min(vecs, 256);
  const int lanes = 256 / cols;
  const int col_in = threadIdx.x % cols, lane = threadIdx.x / cols;
  const int cv = blockIdx.y * cols + col_in;
  if (cv >= vecs || lane >= lanes) return;
  float inv_n;
  if constexpr (std::is_same<S, double>::value)
    inv_n = 1.0f / (float)*n_all;
  else
    inv_n = 1.0f / (float)npix;
  float sc[8], sh[8], k2[8], k3[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = cv * 8 + k;
    sc[k] = scale[c];
    sh[k] = shift[c];
    const float b = invstd[c] * (float)sum_dux[c] * inv_n;
    k2[k] = -sc[k] * b;
    k3[k] = sc[k] * (mean[c] * b - (float)sum_du[c] * inv_n);
  }
  const long long step = (long long)gridDim.x * lanes;
  for (long long p = (long long)blockIdx.x * lanes + lane; p < npix; p += 2 * step) {
    const long long p2 = p + step;
    const bool two = p2 < npix;
    const uint4 z0 = *reinterpret_cast<const uint4*>(z + p * z_stride + cv * 8);
    const uint4 d0 = *reinterpret_cast<const uint4*>(dy + p * dy_stride + cv * 8);
    uint4 z1 = make_uint4(0, 0, 0, 0), d1 = z1, g0 = z1, g1 = z1;
    if (two) {
      z1 = *reinterpret_cast<const uint4*>(z + p2 * z_stride + cv * 8);
      d1 = *reinterpret_cast<const uint4*>(dy + p2 * dy_stride + cv * 8);
    }
    if (gres && gres_accumulate) {
      g0 = *reinterpret_cast<const uint4*>(gres + p * gres_stride + cv * 8);
      if (two) g1 = *reinterpret_cast<const uint4*>(gres + p2 * gres_stride + cv * 8);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1 && !two) break;
      const long long q = h ? p2 : p;
      const uint4 dyv = h ? d1 : d0;
      float zf[8], df[8], o[8];
      unpack8(h ? z1 : z0, zf);
      unpack8(dyv, df);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float du = act ? df[k] * silu_grad(fmaf(zf[k], sc[k], sh[k])) : df[k];
        o[k] = fmaf(sc[k], du, fmaf(k2[k], zf[k], k3[k]));
      }
      *reinterpret_cast<uint4*>(dz + q * dz_stride + cv * 8) = pack8(o);
      if (gres) {
        __nv_bfloat16* g = gres + q * gres_stride + cv * 8;
        if (gres_accumulate) {
          float a[8];
          unpack8(h ? g1 : g0, a);
#pragma unroll
          for (int k = 0; k < 8; ++k) a[k] += df[k];
          *reinterpret_cast<uint4*>(g) = pack8(a);
        } else {
          *reinterpret_cast<uint4*>(g) = dyv;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_bn_bwd_apply(const __nv_bfloat16* __restrict__ z, long long z_stride,
                                                      const __nv_bfloat16* __restrict__ dy, long long dy_stride, long long npix,
                                                      int C, const float* __restrict__ scale, const float* __restrict__ shift,
                                                      const float* __restrict__ mean, const float* __restrict__ invstd, int act,
                                                      const float* __restrict__ sum_du, const float* __restrict__ sum_dux,
                                                      __nv_bfloat16* __restrict__ dz, long long dz_stride,
                                                      __nv_bfloat16* __restrict__ gres, long long gres_stride,
                                                      int gres_accumulate) {
  bn_bwd_apply(z, z_stride, dy, dy_stride, npix, C, scale, shift, mean, invstd, act, sum_du, sum_dux, nullptr, dz, dz_stride,
               gres, gres_stride, gres_accumulate);
}

// SyncBatchNorm backward, second half: rec = [sum(du) | sum(du * xhat)] summed over every rank, n_all = the summed forward
// record's count
__global__ void __launch_bounds__(256) k_bn_bwd_apply_rec(const __nv_bfloat16* __restrict__ z, long long z_stride,
                                                          const __nv_bfloat16* __restrict__ dy, long long dy_stride,
                                                          long long npix, int C, const float* __restrict__ scale,
                                                          const float* __restrict__ shift, const float* __restrict__ mean,
                                                          const float* __restrict__ invstd, int act,
                                                          const double* __restrict__ rec, const double* __restrict__ n_all,
                                                          __nv_bfloat16* __restrict__ dz, long long dz_stride,
                                                          __nv_bfloat16* __restrict__ gres, long long gres_stride,
                                                          int gres_accumulate) {
  bn_bwd_apply(z, z_stride, dy, dy_stride, npix, C, scale, shift, mean, invstd, act, rec, rec + C, n_all, dz, dz_stride, gres,
               gres_stride, gres_accumulate);
}

// gdst[b,h,w,:] (+)= sum of the 2x2 block gsrc[b,2h+{0,1},2w+{0,1},:]   (backward of nn.Upsample(2x nearest))
__global__ void k_upsample2x_bwd(const __nv_bfloat16* __restrict__ gsrc, long long src_stride,
                                 __nv_bfloat16* __restrict__ gdst, long long dst_stride, long long npix, int C, int W,
                                 int accumulate) {
  const int vecs = C >> 3;
  const long long total = npix * vecs;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / vecs;
    const int cv = (int)(i - p * vecs);
    const long long row = p / W;
    const int w = (int)(p - row * W);
    const __nv_bfloat16* s0 = gsrc + ((row * 2) * (2LL * W) + 2 * w) * src_stride + cv * 8;
    float a[8], t[8];
    unpack8(*reinterpret_cast<const uint4*>(s0), a);
    unpack8(*reinterpret_cast<const uint4*>(s0 + src_stride), t);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += t[k];
    unpack8(*reinterpret_cast<const uint4*>(s0 + 2LL * W * src_stride), t);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += t[k];
    unpack8(*reinterpret_cast<const uint4*>(s0 + 2LL * W * src_stride + src_stride), t);
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] += t[k];
    __nv_bfloat16* d = gdst + p * dst_stride + cv * 8;
    if (accumulate) {
      unpack8(*reinterpret_cast<const uint4*>(d), t);
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] += t[k];
    }
    *reinterpret_cast<uint4*>(d) = pack8(a);
  }
}

// one 5x5/s1/p2 max-pool backward step: gin[argmax window position] += gout (first maximum in row-major window order,
// as ATen's max_pool2d_with_indices picks); fp32 accumulation buffer gin32 [npix][C]
__global__ void k_maxpool5_bwd(const __nv_bfloat16* __restrict__ xin, long long in_stride, const float* __restrict__ gout32,
                               const __nv_bfloat16* __restrict__ gout16, long long gout_stride, float* __restrict__ gin32,
                               int B, int H, int W, int C) {
  const long long total = (long long)B * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    long long r = i / C;
    const int w = (int)(r % W);
    r /= W;
    const int h = (int)(r % H);
    const int b = (int)(r / H);
    const long long pix = ((long long)b * H + h) * W + w;
    float g = gout16 ? __bfloat162float(gout16[pix * gout_stride + c]) : 0.f;
    if (gout32) g += gout32[pix * C + c];
    if (g == 0.f) continue;
    float best = -INFINITY;
    long long bp = -1;
    for (int dy = -2; dy <= 2; ++dy) {
      const int hh = h + dy;
      if (hh < 0 || hh >= H) continue;
      for (int dx = -2; dx <= 2; ++dx) {
        const int ww = w + dx;
        if (ww < 0 || ww >= W) continue;
        const long long q = ((long long)b * H + hh) * W + ww;
        const float v = __bfloat162float(xin[q * in_stride + c]);
        if (v > best) {
          best = v;
          bp = q;
        }
      }
    }
    if (bp >= 0) atomicAdd(gin32 + bp * C + c, g);
  }
}

// bf16 slice (+)= fp32 dense
__global__ void k_add_f32_to_bf16(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long dst_stride,
                                  long long npix, int C, int accumulate) {
  const long long total = npix * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / C;
    const int c = (int)(i - p * C);
    __nv_bfloat16* d = dst + p * dst_stride + c;
    const float v = src[i] + (accumulate ? __bfloat162float(*d) : 0.f);
    *d = __float2bfloat16(v);
  }
}

// Detect: loss gradient fp32 [B, na, H, W, no] -> bf16 NHWC [B, H, W, na * bn] (anchor a at channels [a*bn, a*bn + no)),
// four channels per thread (no and bn are multiples of 4)
__global__ void k_detect_grad_pack(const float* __restrict__ g, __nv_bfloat16* __restrict__ out, int B, int na, int H, int W,
                                   int no, int bn) {
  const int q4 = bn >> 2;
  const long long total = (long long)B * H * W * na * q4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % q4) * 4;
    long long r = i / q4;
    const int a = (int)(r % na);
    r /= na;  // pixel index (b * H + h) * W + w
    const long long hw = (long long)H * W;
    const long long b = r / hw, pix = r - b * hw;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < no) v = *reinterpret_cast<const float4*>(g + (((b * na + a) * hw) + pix) * no + c);
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(out + i * 4) = o;
  }
}

// grid of the column-persistent element-wise kernels: x = pixel blocks (two pixels per thread step, <= 8 blocks per SM),
// y = groups of 256 vector columns
dim3 colwise_grid(long long npix, int C) {
  const int vecs = C / 8;
  const int cols = std::min(vecs, 256);
  const int lanes = 256 / cols;
  const long long want = (npix + 2LL * lanes - 1) / (2LL * lanes);
  const int gx = (int)std::max<long long>(1, std::min<long long>(want, (long long)sm_count() * 8));
  return dim3((unsigned)gx, (unsigned)((vecs + cols - 1) / cols), 1);
}

// general (any no) one-channel-per-thread form
__global__ void k_detect_grad_pack1(const float* __restrict__ g, __nv_bfloat16* __restrict__ out, int B, int na, int H, int W,
                                    int no, int bn) {
  const long long total = (long long)B * H * W * na * bn;
  const long long hw = (long long)H * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % bn);
    long long r = i / bn;
    const int a = (int)(r % na);
    r /= na;
    const long long b = r / hw, pix = r - b * hw;
    out[i] = __float2bfloat16(c < no ? g[(((b * na + a) * hw) + pix) * no + c] : 0.f);
  }
}

int stat_blocks_max() { return sm_count() * 4; }
// blocks of the two-stage reductions: >= 16 pixels per thread, at most 4 blocks per SM (every block adds a partial row)
int stat_blocks(long long npix, int C) {
  const int vecs = C / 8;
  const int cols = std::min(vecs, STAT_THREADS);
  const int lanes = STAT_THREADS / cols;
  const long long want = (npix + (long long)lanes * 16 - 1) / ((long long)lanes * 16);
  return (int)std::max<long long>(1, std::min<long long>(want, stat_blocks_max()));
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int64_t y5obb_bn_scratch_floats(int C) { return C > 0 ? (int64_t)stat_blocks_max() * 2 * C : 0; }

int y5obb_bn_stats(const void* z, int64_t z_pix_stride, int64_t npix, int C, float* sum, float* sumsq, float* scratch,
                   int64_t scratch_floats, void* stream) {
  if (!z || !sum || !sumsq || !scratch || npix <= 0 || C <= 0 || (C & 7) || (z_pix_stride & 7)) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(scratch)) & 15) return Y5OBB_EINVAL;
  const int blocks = stat_blocks(npix, C);
  if (scratch_floats < (int64_t)blocks * 2 * C) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long chunk = (npix + blocks - 1) / blocks;
  k_bn_stats<<<blocks, STAT_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride, npix, C, chunk, scratch);
  Y5_LAUNCH_CHECK();
  k_reduce_partials<<<(2 * C + 7) / 8, 256, 0, st>>>(scratch, blocks, C, sum, sumsq, nullptr, nullptr, 0);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_batch_stats(const void* z, int64_t z_pix_stride, int64_t npix, int C, const float* gamma, const float* beta,
                         float eps, float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                         float* mean_out, float* invstd_out, float* scratch, int64_t scratch_floats, void* stream) {
  if (!z || !gamma || !beta || !scale || !shift || !mean_out || !invstd_out || !scratch || npix <= 0 || C <= 0 || (C & 7) ||
      (z_pix_stride & 7))
    return Y5OBB_EINVAL;
  if ((running_mean == nullptr) != (running_var == nullptr)) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(scratch)) & 15) return Y5OBB_EINVAL;
  const int blocks = stat_blocks(npix, C);
  if (scratch_floats < (int64_t)blocks * 2 * C) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long chunk = (npix + blocks - 1) / blocks;
  k_bn_stats<<<blocks, STAT_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride, npix, C, chunk, scratch);
  Y5_LAUNCH_CHECK();
  k_reduce_finalize<<<(C + 7) / 8, 256, 0, st>>>(scratch, blocks, npix, C, gamma, beta, eps, momentum, running_mean,
                                                 running_var, scale, shift, mean_out, invstd_out);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_finalize(const float* sum, const float* sumsq, int64_t npix, int C, const float* gamma, const float* beta,
                      float eps, float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                      float* mean_out, float* invstd_out, void* stream) {
  if (!sum || !sumsq || !gamma || !beta || !scale || !shift || !mean_out || !invstd_out || npix <= 0 || C <= 0)
    return Y5OBB_EINVAL;
  if ((running_mean == nullptr) != (running_var == nullptr)) return Y5OBB_EINVAL;
  k_bn_finalize<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sum, sumsq, npix, C, gamma, beta, eps, momentum,
                                                                    running_mean, running_var, scale, shift, mean_out,
                                                                    invstd_out);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_silu_apply(const void* z, int64_t z_pix_stride, int64_t npix, int C, int W, const float* scale,
                        const float* shift, int act, const void* res, int64_t res_pix_stride, void* y,
                        int64_t y_pix_stride, void* y2x, int64_t y2x_pix_stride, void* stream) {
  if (!z || !scale || !shift || !y || npix <= 0 || C <= 0 || (C & 7) || W <= 0) return Y5OBB_EINVAL;
  if ((z_pix_stride & 7) || (y_pix_stride & 7) || (res && (res_pix_stride & 7)) || (y2x && (y2x_pix_stride & 7)))
    return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(res) |
       reinterpret_cast<uintptr_t>(y2x) | reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift)) & 15)
    return Y5OBB_EINVAL;
  if (y2x && npix % W) return Y5OBB_EINVAL;
  const dim3 grid = colwise_grid(npix, C);
  k_bn_silu_apply<<<grid, 256, 0, (cudaStream_t)stream>>>(
      static_cast<const __nv_bfloat16*>(z), z_pix_stride, npix, C, W, scale, shift, act,
      static_cast<const __nv_bfloat16*>(res), res_pix_stride, static_cast<__nv_bfloat16*>(y), y_pix_stride,
      static_cast<__nv_bfloat16*>(y2x), y2x_pix_stride);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}


int y5obb_bn_silu_bwd(const void* z, int64_t z_pix_stride, const void* dy, int64_t dy_pix_stride, int64_t npix, int C,
                      const float* scale, const float* shift, const float* mean, const float* invstd, int act,
                      float* sum_du, float* sum_dux, void* dz, int64_t dz_pix_stride, void* gres,
                      int64_t gres_pix_stride, int gres_accumulate, float* dgamma, float* dbeta, int param_accumulate,
                      float* scratch, int64_t scratch_floats, void* stream) {
  if ((dgamma == nullptr) != (dbeta == nullptr)) return Y5OBB_EINVAL;
  if (!z || !dy || !scale || !shift || !mean || !invstd || !sum_du || !sum_dux || !dz || !scratch || npix <= 0 || C <= 0 ||
      (C & 7))
    return Y5OBB_EINVAL;
  if ((z_pix_stride & 7) || (dy_pix_stride & 7) || (dz_pix_stride & 7) || (gres && (gres_pix_stride & 7))) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dz) |
       reinterpret_cast<uintptr_t>(gres) | reinterpret_cast<uintptr_t>(scratch)) & 15)
    return Y5OBB_EINVAL;
  const int blocks = stat_blocks(npix, C);
  if (scratch_floats < (int64_t)blocks * 2 * C) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long chunk = (npix + blocks - 1) / blocks;
  k_bn_bwd_reduce<<<blocks, STAT_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride,
                                                   static_cast<const __nv_bfloat16*>(dy), dy_pix_stride, npix, C, scale,
                                                   shift, mean, invstd, act, chunk, scratch);
  Y5_LAUNCH_CHECK();
  k_reduce_partials<<<(2 * C + 7) / 8, 256, 0, st>>>(scratch, blocks, C, sum_du, sum_dux, dgamma, dbeta, param_accumulate);
  Y5_LAUNCH_CHECK();
  const dim3 g2 = colwise_grid(npix, C);
  k_bn_bwd_apply<<<g2, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride,
                                     static_cast<const __nv_bfloat16*>(dy), dy_pix_stride, npix, C, scale, shift, mean,
                                     invstd, act, sum_du, sum_dux, static_cast<__nv_bfloat16*>(dz), dz_pix_stride,
                                     static_cast<__nv_bfloat16*>(gres), gres_pix_stride, gres_accumulate);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_stats_sync(const void* z, int64_t z_pix_stride, int64_t npix, int C, double* rec, float* scratch,
                        int64_t scratch_floats, void* stream) {
  if (!z || !rec || !scratch || npix <= 0 || C <= 0 || (C & 7) || (z_pix_stride & 7)) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(scratch)) & 15) return Y5OBB_EINVAL;
  const int blocks = stat_blocks(npix, C);
  if (scratch_floats < (int64_t)blocks * 2 * C) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long chunk = (npix + blocks - 1) / blocks;
  k_bn_stats<<<blocks, STAT_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride, npix, C, chunk, scratch);
  Y5_LAUNCH_CHECK();
  k_reduce_stats_rec<<<(C + 7) / 8, 256, 0, st>>>(scratch, blocks, npix, C, rec);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_finalize_sync(const double* rec, int C, const float* gamma, const float* beta, float eps, float momentum,
                           float* running_mean, float* running_var, float* scale, float* shift, float* mean_out,
                           float* invstd_out, void* stream) {
  if (!rec || !gamma || !beta || !scale || !shift || !mean_out || !invstd_out || C <= 0) return Y5OBB_EINVAL;
  if ((running_mean == nullptr) != (running_var == nullptr)) return Y5OBB_EINVAL;
  k_bn_finalize_rec<<<(C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(rec, C, gamma, beta, eps, momentum, running_mean,
                                                                        running_var, scale, shift, mean_out, invstd_out);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_silu_bwd_reduce_sync(const void* z, int64_t z_pix_stride, const void* dy, int64_t dy_pix_stride, int64_t npix,
                                  int C, const float* scale, const float* shift, const float* mean, const float* invstd,
                                  int act, double* rec, float* dgamma, float* dbeta, int param_accumulate, float* scratch,
                                  int64_t scratch_floats, void* stream) {
  if ((dgamma == nullptr) != (dbeta == nullptr)) return Y5OBB_EINVAL;
  if (!z || !dy || !scale || !shift || !mean || !invstd || !rec || !scratch || npix <= 0 || C <= 0 || (C & 7))
    return Y5OBB_EINVAL;
  if ((z_pix_stride & 7) || (dy_pix_stride & 7)) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(scratch)) & 15)
    return Y5OBB_EINVAL;
  const int blocks = stat_blocks(npix, C);
  if (scratch_floats < (int64_t)blocks * 2 * C) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const long long chunk = (npix + blocks - 1) / blocks;
  k_bn_bwd_reduce<<<blocks, STAT_THREADS, 0, st>>>(static_cast<const __nv_bfloat16*>(z), z_pix_stride,
                                                   static_cast<const __nv_bfloat16*>(dy), dy_pix_stride, npix, C, scale,
                                                   shift, mean, invstd, act, chunk, scratch);
  Y5_LAUNCH_CHECK();
  k_reduce_partials_rec<<<(2 * C + 7) / 8, 256, 0, st>>>(scratch, blocks, C, rec, dgamma, dbeta, param_accumulate);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_bn_silu_bwd_apply_sync(const void* z, int64_t z_pix_stride, const void* dy, int64_t dy_pix_stride, int64_t npix,
                                 int C, const float* scale, const float* shift, const float* mean, const float* invstd,
                                 int act, const double* rec, const double* n_all, void* dz, int64_t dz_pix_stride,
                                 void* gres, int64_t gres_pix_stride, int gres_accumulate, void* stream) {
  if (!z || !dy || !scale || !shift || !mean || !invstd || !rec || !n_all || !dz || npix <= 0 || C <= 0 || (C & 7))
    return Y5OBB_EINVAL;
  if ((z_pix_stride & 7) || (dy_pix_stride & 7) || (dz_pix_stride & 7) || (gres && (gres_pix_stride & 7))) return Y5OBB_EINVAL;
  if ((reinterpret_cast<uintptr_t>(z) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dz) |
       reinterpret_cast<uintptr_t>(gres)) & 15)
    return Y5OBB_EINVAL;
  const dim3 g2 = colwise_grid(npix, C);
  k_bn_bwd_apply_rec<<<g2, 256, 0, (cudaStream_t)stream>>>(
      static_cast<const __nv_bfloat16*>(z), z_pix_stride, static_cast<const __nv_bfloat16*>(dy), dy_pix_stride, npix, C, scale,
      shift, mean, invstd, act, rec, n_all, static_cast<__nv_bfloat16*>(dz), dz_pix_stride, static_cast<__nv_bfloat16*>(gres),
      gres_pix_stride, gres_accumulate);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_upsample2x_bwd(const void* gsrc, int64_t src_pix_stride, void* gdst, int64_t dst_pix_stride, int64_t npix_dst,
                         int C, int W_dst, int accumulate, void* stream) {
  if (!gsrc || !gdst || npix_dst <= 0 || C <= 0 || (C & 7) || W_dst <= 0 || (src_pix_stride & 7) || (dst_pix_stride & 7))
    return Y5OBB_EINVAL;
  const long long total = npix_dst * (C / 8);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_upsample2x_bwd<<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const __nv_bfloat16*>(gsrc), src_pix_stride,
                                                           static_cast<__nv_bfloat16*>(gdst), dst_pix_stride, npix_dst, C,
                                                           W_dst, accumulate);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_maxpool5_bwd(const void* x_in, int64_t in_pix_stride, const float* gout_f32, const void* gout_bf16,
                       int64_t gout_pix_stride, float* gin_f32, int B, int H, int W, int C, void* stream) {
  if (!x_in || !gin_f32 || (!gout_f32 && !gout_bf16) || B <= 0 || H <= 0 || W <= 0 || C <= 0) return Y5OBB_EINVAL;
  const long long total = (long long)B * H * W * C;
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_maxpool5_bwd<<<grid, 256, 0, (cudaStream_t)stream>>>(static_cast<const __nv_bfloat16*>(x_in), in_pix_stride, gout_f32,
                                                         static_cast<const __nv_bfloat16*>(gout_bf16), gout_pix_stride,
                                                         gin_f32, B, H, W, C);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_add_f32_to_bf16(const float* src, void* dst, int64_t dst_pix_stride, int64_t npix, int C, int accumulate,
                          void* stream) {
  if (!src || !dst || npix <= 0 || C <= 0) return Y5OBB_EINVAL;
  const long long total = npix * C;
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  k_add_f32_to_bf16<<<grid, 256, 0, (cudaStream_t)stream>>>(src, static_cast<__nv_bfloat16*>(dst), dst_pix_stride, npix, C,
                                                            accumulate);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

int y5obb_detect_grad_pack(const float* g, void* out_nhwc, int B, int na, int H, int W, int no, int bn, void* stream) {
  if (!g || !out_nhwc || B <= 0 || na <= 0 || H <= 0 || W <= 0 || no <= 0 || bn < no) return Y5OBB_EINVAL;
  const bool vec4 = !(no & 3) && !(bn & 3) && !(reinterpret_cast<uintptr_t>(g) & 15) && !(reinterpret_cast<uintptr_t>(out_nhwc) & 7);
  const long long total = (long long)B * H * W * na * (vec4 ? bn / 4 : bn);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 16);
  if (vec4)
    k_detect_grad_pack<<<grid, 256, 0, (cudaStream_t)stream>>>(g, static_cast<__nv_bfloat16*>(out_nhwc), B, na, H, W, no, bn);
  else
    k_detect_grad_pack1<<<grid, 256, 0, (cudaStream_t)stream>>>(g, static_cast<__nv_bfloat16*>(out_nhwc), B, na, H, W, no, bn);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

}  // extern "C"
