// Implicit-GEMM NHWC bf16 convolution for sm_90a: TMA -> shared memory -> wgmma (fp32 accumulators in registers) ->
// fused epilogue (folded-BN bias, SiLU, residual add, concat-offset store, 2x nearest up-sample copy, or the Detect
// head's permute + sigmoid + grid/anchor decode).
//
// Replaces, for the layers of models/yolov5{n,s,m,l,x}.yaml, the cuDNN/ATen calls behind
//   models/common.py  Conv.forward_fuse (conv + bias + SiLU), Bottleneck (x + cv2(cv1(x))) -> residual epilogue,
//                     Concat -> channel-offset store
//   models/yolo.py    Detect (1x1 conv, view/permute, sigmoid, decode)
//
// GEMM view: D[128 output pixels, BN channels] = sum over (tap, 64-channel chunk) A_tap[128, BK] * W_tap[BN, BK]^T
//   A tile  = one 4-D TMA box {BK ch, Wt, Ht, 1} of the NHWC input at the tap's shifted origin; zero
//             padding, ragged channel counts and ragged image edges are TMA out-of-bounds zero fill;
//             stride-2 convs use the tensor map's element strides (or the pixel-pair view).
//   W tile  = 2-D TMA box {BK, NI} of weights packed [tap][Cout_pad][Cin_pad] (K-major).
//   Both land in 32/64/128-byte swizzled K-major layouts that wgmma reads through shared-memory descriptors.
// One persistent CTA per SM, three warpgroups: two consumers (pixel rows 0-63 and 64-127 of the tile, each issuing
// m64nNIk16 wgmma over the whole N tile and running the epilogue of its rows) and a producer whose first warp issues the
// TMA loads.  setmaxnreg moves the producer's registers to the consumers (up to 128 fp32 accumulators per thread).  The producer
// runs ahead through a ring of pipeline stages, so the next tile's operands arrive while the epilogue of this one runs.
//
// Roofline: tensor pipe for the wide layers (2*128*BN*K flop per tile), HBM for the narrow ones
// (algorithmic bytes = input pixels*Cin*2 + output pixels*Cout*2 [+ residual] per image).
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

constexpr int BM = 128;  // output pixels per tile
constexpr int MAX_STAGES = 16;
constexpr int CONSUMER_WARPS = 8;                        // two warpgroups of 64 pixel rows each
constexpr int NUM_THREADS = 32 * (CONSUMER_WARPS + 4);   // + the producer warpgroup (one warp issues the TMA loads)
constexpr int STG_PITCH = 68;                            // fp32 per staged row: 64 columns + 4 (spreads the banks)
constexpr int STG_BYTES = (16 * STG_PITCH + 16) * 4;     // per consumer warp: 16 rows x 64 columns, then 16 theta indices
constexpr int SMEM_TOTAL = 224 * 1024;                   // dynamic shared memory we ask for at most (227 KB is the H100 cap)

enum Mode : int { MODE_CONV = 0, MODE_DETECT = 1 };

// division by a launch-time constant without the ~100-cycle integer divide (x < 2^31): q = (umulhi(x, m) + x) >> s
struct FastDiv {
  uint32_t d, m, s;
};
inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  f.d = d;
  uint32_t s = 0;
  while ((1u << s) < d) ++s;
  f.s = s;
  f.m = (uint32_t)((((uint64_t)1 << 32) * (((uint64_t)1 << s) - d)) / d + 1);
  return f;
}
__device__ __forceinline__ uint32_t fdiv(uint32_t x, const FastDiv& f) { return (__umulhi(x, f.m) + x) >> f.s; }

struct ConvK {
  CUtensorMap tmA;
  CUtensorMap tmB;
  // geometry
  int B, Hout, Wout;
  int Wt, Ht, tiles_w, tiles_h;
  int n_tiles_m, n_tiles_n;
  FastDiv fd_ntn, fd_per_img, fd_tiles_w, fd_wt;
  int BN, BK, NI;      // N tile, K chunk, wgmma N (BN rounded up to an instruction shape; extra columns are never stored)
  int Cout, cout_pad;
  int Cin, kchunks, KH, KW, stride, pad_h, pad_w;
  int stages;
  int pdl;             // launched with programmatic stream serialisation: griddepcontrol.wait before the first global access
  int pairw;           // 1: stride-2 conv whose input is viewed as horizontal pixel PAIRS (2*pix_stride channels per
                       // position): the column phase of a tap is a channel offset, so TMA reads contiguous rows
  int in_pix_stride;
  int rowshift;    // 1: one A stage holds Ht + KH - 1 image rows; the KH taps of a column read it at row offsets
  int b_resident;  // 1: every weight tile stays in shared memory for the whole kernel (loaded once)
  int b_per_stage; // weight tiles streamed with each A unit (0 when resident)
  int group;       // (tap, K-chunk) units per pipeline stage: one mbarrier round trip serves `group` TMA boxes
  int n_units;     // units per tile = (rowshift ? KW : KH*KW) * kchunks
  uint32_t a_bytes, a_tx_bytes, b_bytes, b_stage_bytes, b_res_bytes, row_shift_bytes;
  // epilogue
  int mode, act;
  const float* bias;
  __nv_bfloat16* out;
  long long out_pix_stride, out_row_stride, out_img_stride;
  const __nv_bfloat16* res;
  long long res_pix_stride, res_row_stride, res_img_stride;
  __nv_bfloat16* out2x;
  long long out2x_pix_stride;
  // detect
  float* det_out;
  long long det_rows_per_image, det_row_off;
  int det_no, det_decode;  // det_decode: 0 raw logits, 1 sigmoid + grid/anchor decode, 2 = 1 as compact records (see the epilogue)
  int det_rec_w;           // floats per compact record: (5 + nc + 1) rounded up to 4
  float det_stride;
  float det_anchor[6];
};

struct TileCoord {
  int b, h0, w0, n0, nt;
};

__device__ __forceinline__ TileCoord decode_tile(const ConvK& p, int t) {
  TileCoord c;
  const int mt = (int)fdiv((uint32_t)t, p.fd_ntn);
  c.nt = t - mt * p.n_tiles_n;
  const int per_img = p.tiles_h * p.tiles_w;
  c.b = (int)fdiv((uint32_t)mt, p.fd_per_img);
  const int r = mt - c.b * per_img;
  const int th = (int)fdiv((uint32_t)r, p.fd_tiles_w);
  c.h0 = th * p.Ht;
  c.w0 = (r - th * p.tiles_w) * p.Wt;
  c.n0 = c.nt * p.BN;
  return c;
}

// x * sigmoid(x) = h + h * tanh(h), h = x / 2: one MUFU op (tanh.approx, rel. error ~2^-11) instead of ex2 + rcp
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_fast(float v) { return fmaf(0.5f, tanh_fast(0.5f * v), 0.5f); }

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ uint64_t desc_from(uint32_t lo, uint32_t hi) {
  uint64_t d;
  asm volatile("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}

// ---- epilogue of one tile for one consumer warp ----------------------------------------------------------------------
// The warp owns 16 pixel rows (row0 .. row0 + 15 of the tile).  wgmma's accumulator layout gives thread `lane` the rows
// row0 + lane / 4 (+ 8) and the column pairs 8 j + 2 (lane % 4) (+ 1).  Each 64-column block is activated in registers,
// staged through shared memory as [16 rows][64] fp32 and leaves in 16-byte vectors per pixel.
template <int NI>
__device__ __forceinline__ void epilogue(const ConvK& p, const TileCoord& c, float (&acc)[NI / 2], float* stg, const float* bias_s,
                                         int row0, int lane) {
  const int q = lane & 3, r = lane >> 2;
  float* theta_s = stg + 16 * STG_PITCH;
  const bool det = p.mode == MODE_DETECT;
  const int nvalid = min(p.BN, (det ? p.det_no : p.Cout - c.n0));
  const int nfix = p.det_no - 180;  // Detect: 5 + nc leading columns, then the theta bins
  const float* bias = bias_s + c.n0;
  if (det && p.det_decode == 2) {
    // the theta index of each row: the first maximum of the 180 theta LOGITS (the sigmoid is monotone, so this is the index
    // torch.max returns on the activated values whenever those are distinct)
    float best[2] = {-INFINITY, -INFINITY};
    int bk[2] = {0, 0};
#pragma unroll
    for (int j = 0; j < NI / 8; ++j)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int col = 8 * j + 2 * q + k;
        if (col >= nfix && col < p.det_no) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float v = acc[4 * j + 2 * i + k] + bias[col];
            if (v > best[i]) {
              best[i] = v;
              bk[i] = col - nfix;
            }
          }
        }
      }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best[i], off);
        const int ok = __shfl_xor_sync(0xffffffffu, bk[i], off);
        if (ob > best[i] || (ob == best[i] && ok < bk[i])) {
          best[i] = ob;
          bk[i] = ok;
        }
      }
      if (q == 0) theta_s[r + 8 * i] = (float)bk[i];
    }
  }
  const int ncols = (det && p.det_decode == 2) ? p.det_rec_w : nvalid;  // columns that leave the kernel
#pragma unroll
  for (int cb = 0; cb < NI; cb += 64) {
    if (cb >= ncols) break;
    // (1) bias (+ SiLU) in registers, staged as fp32
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = cb / 8 + jj;
      if (j < NI / 8) {
        const int col = 8 * j + 2 * q;
        const float b0 = bias[col], b1 = bias[col + 1];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
          if (p.act) {  // SiLU(x) = h + h * tanh(h), h = x / 2 = 0.5 * acc + (0.5 * bias)
            const float h0 = fmaf(v0, 0.5f, b0), h1 = fmaf(v1, 0.5f, b1);
            v0 = fmaf(h0, tanh_fast(h0), h0);
            v1 = fmaf(h1, tanh_fast(h1), h1);
          } else {
            v0 += b0;
            v1 += b1;
          }
          *reinterpret_cast<float2*>(stg + (r + 8 * i) * STG_PITCH + (col - cb)) = make_float2(v0, v1);
        }
      }
    }
    __syncwarp();
    // (2) 16 rows x (up to) 64 columns leave in vectors
    if (!det) {
      for (int v = lane; v < 16 * 8; v += 32) {
        const int row = v >> 3, col = cb + (v & 7) * 8;
        const int tr = row0 + row;
        const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
        const int h = c.h0 + hl, w = c.w0 + (tr - hl * p.Wt);
        if (col >= nvalid || h >= p.Hout || w >= p.Wout) continue;
        const float* sp = stg + row * STG_PITCH + (col - cb);
        const float4 x0 = *reinterpret_cast<const float4*>(sp), x1 = *reinterpret_cast<const float4*>(sp + 4);
        float f[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
        const int ch = c.n0 + col;
        if (p.res) {
          const uint4 rv = *reinterpret_cast<const uint4*>(p.res + (long long)c.b * p.res_img_stride + (long long)h * p.res_row_stride +
                                                            (long long)w * p.res_pix_stride + ch);
          const __nv_bfloat162* rh = reinterpret_cast<const __nv_bfloat162*>(&rv);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 g = __bfloat1622float2(rh[k]);
            f[2 * k] += g.x;
            f[2 * k + 1] += g.y;
          }
        }
        uint4 o;
        o.x = pack_bf16(f[0], f[1]);
        o.y = pack_bf16(f[2], f[3]);
        o.z = pack_bf16(f[4], f[5]);
        o.w = pack_bf16(f[6], f[7]);
        *reinterpret_cast<uint4*>(p.out + (long long)c.b * p.out_img_stride + (long long)h * p.out_row_stride +
                                  (long long)w * p.out_pix_stride + ch) = o;
        if (p.out2x) {  // nn.Upsample(2x nearest): the same vector on the four (dy, dx) phases
          const long long px = p.out2x_pix_stride, rw = 2LL * p.Wout * px;
          __nv_bfloat16* u = p.out2x + (((long long)c.b * 2 * p.Hout + 2 * h) * (2 * p.Wout) + 2 * w) * px + ch;
          *reinterpret_cast<uint4*>(u) = o;
          *reinterpret_cast<uint4*>(u + px) = o;
          *reinterpret_cast<uint4*>(u + rw) = o;
          *reinterpret_cast<uint4*>(u + rw + px) = o;
        }
      }
    } else {
      // Detect, N tile nt == anchor nt.  Output row = b * rows_per_image + row_off + (a * H + h) * W + w (models/yolo.py):
      // the permute is the store's addressing.  det_decode 2 writes compact records (cx, cy, w, h, obj, cls[nc], theta
      // index, padding) - everything non_max_suppression_obb reads of a row - instead of the det_no columns.
      const int a = c.nt;
      const int rw = p.det_decode == 2 ? p.det_rec_w : p.det_no;
      for (int v = lane; v < 16 * 16; v += 32) {
        const int row = v >> 4, col = cb + (v & 15) * 4;
        const int tr = row0 + row;
        const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
        const int h = c.h0 + hl, w = c.w0 + (tr - hl * p.Wt);
        if (col >= ncols || h >= p.Hout || w >= p.Wout) continue;
        const float4 x = *reinterpret_cast<const float4*>(stg + row * STG_PITCH + (col - cb));
        float f[4] = {x.x, x.y, x.z, x.w};
        if (p.det_decode) {
#pragma unroll
          for (int k = 0; k < 4; ++k) f[k] = sigmoid_fast(f[k]);
          if (col == 0) {  // xy, wh (models/yolo.py)
            f[0] = (f[0] * 2.0f - 0.5f + (float)w) * p.det_stride;
            f[1] = (f[1] * 2.0f - 0.5f + (float)h) * p.det_stride;
            f[2] = (f[2] * 2.0f) * (f[2] * 2.0f) * p.det_anchor[2 * a];
            f[3] = (f[3] * 2.0f) * (f[3] * 2.0f) * p.det_anchor[2 * a + 1];
          }
          if (p.det_decode == 2) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if (col + k >= nfix) f[k] = col + k == nfix ? theta_s[row] : 0.0f;
          }
        }
        const long long orow = (long long)c.b * p.det_rows_per_image + p.det_row_off + ((long long)a * p.Hout + h) * p.Wout + w;
        *reinterpret_cast<float4*>(p.det_out + orow * rw + col) = make_float4(f[0], f[1], f[2], f[3]);
      }
    }
    __syncwarp();
  }
}

template <int NI>
__global__ void __launch_bounds__(NUM_THREADS, 1) conv_wgmma_kernel(const __grid_constant__ ConvK p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[MAX_STAGES];
  __shared__ __align__(8) uint64_t empty_bar[MAX_STAGES];
  __shared__ __align__(8) uint64_t wres_bar;

  // 1024-byte aligned: [resident weights][operand ring][epilogue staging][bias] (swizzle patterns repeat every 8 rows)
  uint8_t* smem_res = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* smem = smem_res + p.b_res_bytes;
  const uint32_t unit_bytes = p.a_bytes + (uint32_t)p.b_per_stage * p.b_stage_bytes;
  const uint32_t stage_bytes = unit_bytes * (uint32_t)p.group;
  uint8_t* stg_all = smem + (size_t)p.stages * stage_bytes;
  float* bias_s = reinterpret_cast<float*>(stg_all + (size_t)CONSUMER_WARPS * STG_BYTES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int total_tiles = p.n_tiles_m * p.n_tiles_n;
  const int ksub = p.rowshift ? p.KH : 1;  // taps served by one A stage

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&p.tmA);
    ptx::prefetch_tmap(&p.tmB);
    for (int s = 0; s < p.stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], CONSUMER_WARPS);
    }
    ptx::mbar_init(&wres_bar, 1);
    ptx::fence_mbar_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above overlapped the previous kernel's tail; from here on global memory is
  // touched, so the previous grid must have completed and flushed.  Only then may the NEXT kernel start its own prologue.
  if (p.pdl) {
    ptx::griddep_wait();
    ptx::griddep_launch_dependents();
  }

  if (warp >= CONSUMER_WARPS) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == CONSUMER_WARPS && ptx::elect_one()) {
      if (p.b_resident) {  // all weight tiles, once: tile (tap, kc) at smem_res + (tap * kchunks + kc) * b_stage_bytes
        const int ntile = p.KH * p.KW * p.kchunks;
        ptx::mbar_expect_tx(&wres_bar, (uint32_t)ntile * p.b_bytes);
        for (int tap = 0; tap < p.KH * p.KW; ++tap)
          for (int kc = 0; kc < p.kchunks; ++kc)
            ptx::tma_load_2d(smem_res + (size_t)(tap * p.kchunks + kc) * p.b_stage_bytes, &p.tmB, &wres_bar, kc * p.BK,
                             tap * p.cout_pad + (int)(blockIdx.x % (unsigned)p.n_tiles_n) * p.BN);  // this CTA's N tile (see the host plan)
      }
      int s = 0;
      uint32_t ph = 0;
      const uint32_t unit_tx = p.a_tx_bytes + (uint32_t)p.b_per_stage * p.b_bytes;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const TileCoord c = decode_tile(p, t);
        int kh = 0, kw = 0, kc = 0;  // unit = (tap, kc), kc fastest; rowshift: taps = kw only (kh stays 0), else kh * KW + kw
        for (int u0 = 0; u0 < p.n_units; u0 += p.group) {
          const int ng = min(p.group, p.n_units - u0);
          ptx::mbar_wait(&empty_bar[s], ph ^ 1u);
          uint8_t* sbase = smem + (size_t)s * stage_bytes;
          ptx::mbar_expect_tx(&full_bar[s], unit_tx * (uint32_t)ng);
          for (int g = 0; g < ng; ++g) {
            int wi = c.w0 * p.stride + kw - p.pad_w;
            const int hi = c.h0 * p.stride + kh - p.pad_h;
            int cbase = 0;
            if (p.pairw) {  // input column 2*wo + (kw - pad): pair index wo + floor(off / 2), phase off & 1
              const int off = kw - p.pad_w;
              const int phase = off & 1;
              wi = c.w0 + ((off - phase) >> 1);
              cbase = phase * p.in_pix_stride;
            }
            uint8_t* sa = sbase + (size_t)g * unit_bytes;
            uint8_t* sb = sa + p.a_bytes;
            ptx::tma_load_4d(sa, &p.tmA, &full_bar[s], cbase + kc * p.BK, wi, hi, c.b);
            for (int j = 0; j < p.b_per_stage; ++j) {
              const int tap = (p.rowshift ? j : kh) * p.KW + kw;
              ptx::tma_load_2d(sb + (size_t)j * p.b_stage_bytes, &p.tmB, &full_bar[s], kc * p.BK, tap * p.cout_pad + c.n0);
            }
            if (++kc == p.kchunks) {
              kc = 0;
              if (++kw == p.KW) {
                kw = 0;
                ++kh;
              }
            }
          }
          if (++s == p.stages) {
            s = 0;
            ph ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns pixel rows [64 wg, 64 wg + 64) of every tile =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  for (int i = threadIdx.x; i < p.cout_pad + 32; i += 32 * CONSUMER_WARPS) bias_s[i] = __ldg(p.bias + i);
  asm volatile("bar.sync 1, %0;" ::"n"(32 * CONSUMER_WARPS) : "memory");
  if (p.b_resident) ptx::mbar_wait(&wres_bar, 0u);

  const int wg = warp >> 2;
  float* stg = reinterpret_cast<float*>(stg_all + (size_t)warp * STG_BYTES);
  // descriptors differ only in the 14-bit (address >> 4) field of the low word
  const uint64_t desc0 = ptx::make_kmajor_desc(0u, (uint32_t)p.BK * 2u);
  const uint32_t hi = (uint32_t)(desc0 >> 32);
  const uint32_t ring_lo = (uint32_t)desc0 | ((ptx::smem_u32(smem) & 0x3FFFFu) >> 4);
  const uint32_t res_lo = (uint32_t)desc0 | ((ptx::smem_u32(smem_res) & 0x3FFFFu) >> 4);
  const uint32_t stage16 = stage_bytes >> 4, unit16 = unit_bytes >> 4;
  const uint32_t a_step = p.row_shift_bytes >> 4;  // per vertical tap: one image row of the tile ...
  const uint32_t bst16 = p.b_stage_bytes >> 4;
  const uint32_t b_step = p.b_resident ? (uint32_t)(p.KW * p.kchunks) * bst16 : bst16;  // ... and KW weight tiles (resident) or one
  const uint32_t a_bytes16 = p.a_bytes >> 4;
  const uint32_t a_wg16 = (uint32_t)(wg * 64 * p.BK * 2) >> 4;  // this warpgroup's 64 rows of the A tile
  const int kchunks = p.kchunks, n_units = p.n_units, group = p.group, stages = p.stages;
  const int nk_full = (min(p.BK, p.Cin) + 15) >> 4;                    // k16 steps per tap of a full K chunk
  const int nk_last = ((p.Cin - (kchunks - 1) * p.BK) + 15) >> 4;      // ... of the last (possibly ragged) one
  const bool resident = p.b_resident != 0;

  float acc[NI / 2];
#pragma unroll
  for (int i = 0; i < NI / 2; ++i) acc[i] = 0.0f;
  int s = 0, prev_s = -1;
  uint32_t ph = 0, s_lo = ring_lo;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const TileCoord c = decode_tile(p, t);
    uint32_t scale_d = 0u, bres_lo = res_lo;
    int kc = 0;
    for (int u0 = 0; u0 < n_units; u0 += group) {
      const int ng = min(group, n_units - u0);
      ptx::mbar_wait(&full_bar[s], ph);
      ptx::wgmma_fence_regs(acc);
      ptx::wgmma_fence();
      uint32_t u_lo = s_lo;
      for (int g = 0; g < ng; ++g) {
        const uint32_t a_lo = u_lo + a_wg16;
        const uint32_t b_lo = resident ? bres_lo : u_lo + a_bytes16;
        const bool last = kc + 1 == kchunks;
        const int nk = last ? nk_last : nk_full;
        for (int u = 0; u < ksub; ++u)
          for (int j = 0; j < nk; ++j) {
            ptx::Wgmma<NI>::template mma<0, 0>(acc, desc_from(a_lo + (uint32_t)u * a_step + 2u * j, hi),
                                               desc_from(b_lo + (uint32_t)u * b_step + 2u * j, hi), scale_d);
            scale_d = 1u;
          }
        u_lo += unit16;
        bres_lo += bst16;
        kc = last ? 0 : kc + 1;
      }
      ptx::wgmma_commit();
      ptx::wgmma_fence_regs(acc);
      // the previous stage's MMAs have completed once at most this stage's group is pending: hand that stage back
      ptx::wgmma_wait<1>();
      ptx::wgmma_fence_regs(acc);
      if (prev_s >= 0) {
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[prev_s]);
      }
      prev_s = s;
      s_lo += stage16;
      if (++s == stages) {
        s = 0;
        ph ^= 1u;
        s_lo = ring_lo;
      }
    }
    ptx::wgmma_wait<0>();
    ptx::wgmma_fence_regs(acc);
    __syncwarp();
    if (lane == 0) ptx::mbar_arrive(&empty_bar[prev_s]);
    prev_s = -1;
    epilogue<NI>(p, c, acc, stg, bias_s, wg * 64 + (warp & 3) * 16, lane);
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_tmapEncodeTiled get_encode() {
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

CUtensorMapSwizzle swizzle_for(int bk) {
  return bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// wgmma N for an N tile of bn columns: 16, or a multiple of 32
int instr_n(int bn) { return bn <= 16 ? 16 : (bn + 31) / 32 * 32; }

typedef void (*KernelFn)(ConvK);
KernelFn kernel_for(int ni) {
  switch (ni) {
    case 16: return conv_wgmma_kernel<16>;
    case 32: return conv_wgmma_kernel<32>;
    case 64: return conv_wgmma_kernel<64>;
    case 96: return conv_wgmma_kernel<96>;
    case 128: return conv_wgmma_kernel<128>;
    case 160: return conv_wgmma_kernel<160>;
    case 192: return conv_wgmma_kernel<192>;
    case 224: return conv_wgmma_kernel<224>;
    case 256: return conv_wgmma_kernel<256>;
    default: return nullptr;
  }
}

struct ConvObj {
  ConvK k;
  KernelFn fn;
  int grid;
  int threads;
  size_t smem;
  double flops;      // algorithmic 2*MACs
  double hbm_bytes;  // algorithmic in + out (+ residual) bytes
};

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

int y5obb_conv_tiling(int cin, int cout, int mode, int det_no, int* block_k, int* block_n, int* cin_pad,
                      int* cout_pad, int* n_tiles_n) {
  if (cin <= 0 || cout <= 0 || !block_k || !block_n || !cin_pad || !cout_pad || !n_tiles_n) return Y5OBB_EINVAL;
  int bk = cin > 32 ? 64 : (cin > 16 ? 32 : 16);
  int bn, nt;
  if (mode == MODE_DETECT) {
    if (det_no <= 0 || cout % det_no) return Y5OBB_EINVAL;
    nt = cout / det_no;
    bn = (det_no + 15) / 16 * 16;
    if (bn > 256) return Y5OBB_EINVAL;
  } else {
    int best_nt = 0, best_bn = 0;
    long best_cost = -1;
    for (nt = (cout + 255) / 256; nt <= (cout + 255) / 256 + 3; ++nt) {
      bn = ((cout + nt - 1) / nt + 15) / 16 * 16;
      if (bn > 256) continue;
      long cost = (long)bn * nt * 16 + nt;  // padded width first, then fewer tiles
      if (best_cost < 0 || cost < best_cost) {
        best_cost = cost;
        best_nt = nt;
        best_bn = bn;
      }
    }
    nt = best_nt;
    bn = best_bn;
  }
  *block_k = bk;
  *block_n = bn;
  *cin_pad = (cin + 7) / 8 * 8;
  *cout_pad = bn * nt;
  *n_tiles_n = nt;
  return Y5OBB_OK;
}

int y5obb_conv_create(const y5obb_conv_desc* d, y5obb_conv_t** out) {
  if (!d || !out) return Y5OBB_EINVAL;
  if (!d->in || !d->w || !d->bias) return Y5OBB_EINVAL;
  if (d->stride != 1 && d->stride != 2) return Y5OBB_EINVAL;
  if (d->in_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->in) & 15)) return Y5OBB_EINVAL;
  if (d->KH < 1 || d->KW < 1 || d->pad_h < 0 || d->pad_w < 0) return Y5OBB_EINVAL;
  if (d->mode == MODE_CONV && d->act && !(d->flags & Y5OBB_CONV_BIAS_HALVED)) return Y5OBB_EINVAL;
  const int64_t in_row_stride = d->in_row_stride ? d->in_row_stride : d->in_pix_stride * d->Win;
  const int64_t in_img_stride = d->in_img_stride ? d->in_img_stride : in_row_stride * d->Hin;
  if (in_row_stride % 8 || in_img_stride % 8) return Y5OBB_EINVAL;
  PFN_tmapEncodeTiled enc = get_encode();
  if (!enc) return Y5OBB_ECUDA;

  int bk, bn, cin_pad, cout_pad, nt;
  int rc = y5obb_conv_tiling(d->Cin, d->Cout, d->mode, d->det_no, &bk, &bn, &cin_pad, &cout_pad, &nt);
  if (rc) return rc;

  ConvObj* o = new ConvObj();
  ConvK& k = o->k;
  memset(&k, 0, sizeof(k));
  const bool geom = d->out_h > 0 || d->out_w > 0 || d->out_row_stride || d->out_img_stride || d->res_row_stride || d->res_img_stride;
  if (geom && (d->mode != MODE_CONV || d->out2x || d->out_h <= 0 || d->out_w <= 0 || !d->out_row_stride || !d->out_img_stride ||
               (d->res && (!d->res_row_stride || !d->res_img_stride)) || (d->out_row_stride & 7) || (d->out_img_stride & 7) ||
               (d->res_row_stride & 7) || (d->res_img_stride & 7))) {
    delete o;
    return Y5OBB_EINVAL;
  }
  const int Hout = geom ? d->out_h : (d->Hin + 2 * d->pad_h - d->KH) / d->stride + 1;
  const int Wout = geom ? d->out_w : (d->Win + 2 * d->pad_w - d->KW) / d->stride + 1;
  const int ni = instr_n(bn);
  o->fn = kernel_for(ni);
  if (!o->fn) {
    delete o;
    return Y5OBB_EINVAL;
  }
  k.B = d->B;
  k.Hout = Hout;
  k.Wout = Wout;
  k.n_tiles_n = nt;
  k.BN = bn;
  k.BK = bk;
  k.NI = ni;
  k.Cout = d->Cout;
  k.cout_pad = cout_pad;
  k.Cin = d->Cin;
  k.kchunks = (d->Cin + bk - 1) / bk;
  k.KH = d->KH;
  k.KW = d->KW;
  k.stride = d->stride;
  k.pad_h = d->pad_h;
  k.pad_w = d->pad_w;
  k.b_bytes = (uint32_t)ni * bk * 2;  // the weight box has NI rows (rows past the tile feed columns that are never stored)
  k.b_stage_bytes = (uint32_t)align_up(k.b_bytes, 1024);
  int a_rows = 0;
  size_t stage_bytes = 0;
  const size_t bias_bytes = align_up((size_t)(cout_pad + 32) * 4, 128);  // the bias lives in shared memory behind the staging buffers
  const size_t SMEM_BUDGET = (size_t)SMEM_TOTAL - 1024 - (size_t)CONSUMER_WARPS * STG_BYTES - bias_bytes;
  // Row-shift mode (stride-1 convs with KH > 1): an 8 x 16 pixel tile whose A stage holds Ht + KH - 1 image
  // rows; the KH vertical taps read the same stage at row offsets that are whole 8-row swizzle groups, so each
  // input row crosses L2 -> shared memory (Ht + KH - 1) / Ht times per kw instead of KH times.  Taken when the
  // weights are resident or at least 3 pipeline stages still fit; otherwise one load per tap (classic).
  auto plan = [&](bool rowshift) -> bool {
    int best_wt = 128;
    if (rowshift) {
      best_wt = 8;
    } else {  // Wt x Ht = 128 pixels, Wt the power of two (<=128) that wastes the fewest edge pixels
      double best_eff = -1;
      for (int wt = 128; wt >= 8; wt >>= 1) {
        int ht = BM / wt;
        if (wt * d->stride > 256 || ht * d->stride > 256) continue;
        double eff = (double)Wout * Hout / ((double)((Wout + wt - 1) / wt * wt) * ((Hout + ht - 1) / ht * ht));
        if (eff > best_eff + 1e-9) {
          best_eff = eff;
          best_wt = wt;
        }
      }
    }
    k.Wt = best_wt;
    k.Ht = BM / best_wt;
    k.tiles_w = (Wout + k.Wt - 1) / k.Wt;
    k.tiles_h = (Hout + k.Ht - 1) / k.Ht;
    k.n_tiles_m = d->B * k.tiles_w * k.tiles_h;
    k.rowshift = rowshift ? 1 : 0;
    a_rows = rowshift ? k.Ht + d->KH - 1 : k.Ht;  // image rows per A stage
    if (a_rows * d->stride > 256) return false;    // TMA box dimension limit
    k.a_tx_bytes = (uint32_t)a_rows * k.Wt * bk * 2;
    k.row_shift_bytes = (uint32_t)k.Wt * bk * 2;
    const size_t a_stage = align_up(k.a_tx_bytes, 1024);
    k.a_bytes = (uint32_t)a_stage;  // ring slots are 1024-aligned; the TMA box fills the first a_rows * Wt rows
    const size_t b_all = (size_t)d->KH * d->KW * k.kchunks * k.b_stage_bytes;
    // weights stay resident when they leave room for >= 3 A stages and every CTA keeps one N tile (the grid is made a
    // multiple of their count, so that tile t = blockIdx.x + i * gridDim.x keeps ONE N tile per CTA - the Detect head's three
    // anchors - and that tile's weights are the resident ones)
    k.b_resident = (nt <= 4 && b_all + 3 * a_stage <= SMEM_BUDGET && !(d->flags & Y5OBB_CONV_NO_RESIDENT)) ? 1 : 0;
    k.b_res_bytes = k.b_resident ? (uint32_t)b_all : 0u;
    k.b_per_stage = k.b_resident ? 0 : (rowshift ? d->KH : 1);
    const size_t unit_bytes = a_stage + (size_t)k.b_per_stage * k.b_stage_bytes;
    k.n_units = (rowshift ? d->KW : d->KH * d->KW) * k.kchunks;
    // small units share a stage: every mbarrier round trip then moves >= ~24 KB
    int group = 1;
    if (!(d->flags & Y5OBB_CONV_NO_GROUP))
      while (group < k.n_units && group < 4 && (size_t)(group + 1) * unit_bytes <= 40 * 1024 &&
             (SMEM_BUDGET - k.b_res_bytes) / ((size_t)(group + 1) * unit_bytes) >= 3)
        ++group;
    k.group = group;
    stage_bytes = unit_bytes * group;
    k.stages = (int)std::min<size_t>(MAX_STAGES, (SMEM_BUDGET - k.b_res_bytes) / stage_bytes);
    return k.stages >= (rowshift ? 3 : 2);
  };
  const bool want_rowshift = d->stride == 1 && d->KH > 1 && Wout >= 8 && !(d->flags & Y5OBB_CONV_NO_ROWSHIFT);
  if (!((want_rowshift && plan(true)) || plan(false))) {
    delete o;
    return Y5OBB_EINVAL;
  }
  {
    const char* e = getenv("Y5OBB_NO_PDL");
    k.pdl = ((d->flags & Y5OBB_CONV_NO_PDL) || (e && e[0] == '1')) ? 0 : 1;
  }
  k.fd_ntn = make_fastdiv((uint32_t)k.n_tiles_n);
  k.fd_per_img = make_fastdiv((uint32_t)(k.tiles_h * k.tiles_w));
  k.fd_tiles_w = make_fastdiv((uint32_t)k.tiles_w);
  k.fd_wt = make_fastdiv((uint32_t)k.Wt);
  k.mode = d->mode;
  k.act = d->act;
  k.bias = d->bias;
  k.out = static_cast<__nv_bfloat16*>(d->out);
  k.out_pix_stride = d->out_pix_stride;
  k.out_row_stride = geom ? d->out_row_stride : d->out_pix_stride * Wout;
  k.out_img_stride = geom ? d->out_img_stride : d->out_pix_stride * Wout * Hout;
  k.res = static_cast<const __nv_bfloat16*>(d->res);
  k.res_pix_stride = d->res_pix_stride;
  k.res_row_stride = geom ? d->res_row_stride : d->res_pix_stride * Wout;
  k.res_img_stride = geom ? d->res_img_stride : d->res_pix_stride * Wout * Hout;
  k.out2x = static_cast<__nv_bfloat16*>(d->out2x);
  k.out2x_pix_stride = d->out2x_pix_stride;
  k.det_out = d->det_out;
  k.det_rows_per_image = d->det_rows_per_image;
  k.det_row_off = d->det_row_off;
  k.det_no = d->det_no;
  k.det_decode = d->det_decode;
  k.det_rec_w = ((d->det_no - 180 + 1) + 3) / 4 * 4;
  k.det_stride = d->det_stride;
  for (int i = 0; i < 6; ++i) k.det_anchor[i] = d->det_anchor[i];
  if (d->mode == MODE_CONV) {
    if (!d->out || d->out_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->out) & 15) || d->Cout % 8 ||
        (d->res && (d->res_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->res) & 15))) ||
        (d->out2x && (d->out2x_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->out2x) & 15)))) {
      delete o;
      return Y5OBB_EINVAL;
    }
  } else {
    const int rw = d->det_decode == 2 ? k.det_rec_w : d->det_no;
    if (!d->det_out || d->det_no % 4 || (d->det_decode == 2 && d->det_no <= 180) ||
        (reinterpret_cast<uintptr_t>(d->det_out + (size_t)d->det_row_off * rw) & 15)) {
      delete o;
      return Y5OBB_EINVAL;
    }
  }

  // stride-2 convs over dense rows: view the input as horizontal pixel pairs so that no element stride is needed
  // along W (channels beyond the slice are finite activations of the same buffer and meet zero weights)
  k.pairw = (d->stride == 2 && !(d->Win & 1) && in_row_stride == d->in_pix_stride * d->Win &&
             !(d->flags & Y5OBB_CONV_NO_PAIRW)) ? 1 : 0;
  k.in_pix_stride = (int)d->in_pix_stride;
  {  // activations: (C, W, H, B), element strides (1, s, s, 1)
    cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->Win, (cuuint64_t)d->Hin, (cuuint64_t)d->B};
    cuuint64_t strides[3] = {(cuuint64_t)d->in_pix_stride * 2, (cuuint64_t)in_row_stride * 2,
                             (cuuint64_t)in_img_stride * 2};
    cuuint32_t box[4] = {(cuuint32_t)bk, (cuuint32_t)(k.Wt * d->stride), (cuuint32_t)(a_rows * d->stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
    if (k.pairw) {
      dims[0] = (cuuint64_t)d->in_pix_stride + d->Cin;
      dims[1] = (cuuint64_t)d->Win / 2;
      strides[0] = (cuuint64_t)d->in_pix_stride * 4;
      box[1] = (cuuint32_t)k.Wt;
      es[1] = 1;
    }
    CUresult r = enc(&k.tmA, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->in), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(bk), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      g_last_cuda_error = (int)r;
      delete o;
      return Y5OBB_ECUDA;
    }
  }
  {  // weights: (Cin, taps * Cout_pad)
    cuuint64_t dims[2] = {(cuuint64_t)d->Cin, (cuuint64_t)d->KH * d->KW * cout_pad};
    cuuint64_t strides[1] = {(cuuint64_t)cin_pad * 2};
    cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)ni};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&k.tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d->w), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(bk), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      g_last_cuda_error = (int)r;
      delete o;
      return Y5OBB_ECUDA;
    }
  }
  const int total = k.n_tiles_m * k.n_tiles_n;
  o->grid = std::min(total, sm_count());
  if (k.b_resident && k.n_tiles_n > 1) o->grid = o->grid / k.n_tiles_n * k.n_tiles_n;  // one N tile per CTA (resident weights)
  o->threads = NUM_THREADS;
  o->smem = k.b_res_bytes + (size_t)k.stages * stage_bytes + (size_t)CONSUMER_WARPS * STG_BYTES + bias_bytes + 1024;
  o->flops = 2.0 * d->B * Hout * Wout * (double)d->Cout * d->Cin * d->KH * d->KW;
  o->hbm_bytes = 2.0 * d->B * ((double)d->Hin * d->Win * (d->hbm_cin ? d->hbm_cin : d->Cin) + (double)Hout * Wout * d->Cout * (d->res ? 2 : 1));
  static bool attr_set[257] = {};
  if (!attr_set[ni]) {
    cudaError_t e = cudaFuncSetAttribute(o->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL);
    if (e != cudaSuccess) {
      delete o;
      return cuda_fail(e);
    }
    attr_set[ni] = true;
  }
  *out = reinterpret_cast<y5obb_conv_t*>(o);
  return Y5OBB_OK;
}

int y5obb_conv_run(const y5obb_conv_t* conv, void* stream) {
  if (!conv) return Y5OBB_EINVAL;
  const ConvObj* o = reinterpret_cast<const ConvObj*>(conv);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)o->grid);
  cfg.blockDim = dim3((unsigned)o->threads);
  cfg.dynamicSmemBytes = o->smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = o->k.pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, o->fn, o->k);
  if (e != cudaSuccess) return cuda_fail(e);
  return Y5OBB_OK;
}

int y5obb_conv_info(const y5obb_conv_t* conv, double* flops, double* hbm_bytes, int* grid, int* block_n, int* block_k,
                    int* stages) {
  if (!conv) return Y5OBB_EINVAL;
  const ConvObj* o = reinterpret_cast<const ConvObj*>(conv);
  if (flops) *flops = o->flops;
  if (hbm_bytes) *hbm_bytes = o->hbm_bytes;
  if (grid) *grid = o->grid;
  if (block_n) *block_n = o->k.BN;
  if (block_k) *block_k = o->k.BK;
  if (stages) *stages = o->k.stages;
  return Y5OBB_OK;
}

void y5obb_conv_destroy(y5obb_conv_t* conv) { delete reinterpret_cast<ConvObj*>(conv); }

}  // extern "C"
