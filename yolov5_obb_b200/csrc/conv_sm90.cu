// Implicit-GEMM NHWC bf16 (or fp16, F16 / Y5OBB_CONV_F16) convolution for sm_90a: TMA -> shared memory -> wgmma (fp32 accumulators in registers) ->
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
// Persistent CTAs (one per SM, or two for N tiles <= 96, see Occupancy), three warpgroups: two consumers (pixel rows 0-63 and 64-127 of the tile, each issuing
// m64nNIk16 wgmma over the whole N tile and running the epilogue of its rows) and a producer whose first warp issues the
// TMA loads.  setmaxnreg moves the producer's registers to the consumers (up to 128 fp32 accumulators per thread).  The producer
// runs ahead through a ring of pipeline stages, so the next tile's operands arrive while the epilogue of this one runs.
//
// Roofline: tensor pipe for the wide layers (2*128*BN*K flop per tile), HBM for the narrow ones
// (algorithmic bytes = input pixels*Cin*2 + output pixels*Cout*2 [+ residual] per image).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

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
constexpr int SMEM_TOTAL = 224 * 1024;                   // dynamic shared memory we ask for at most (227 KB is the H100 cap)
// Two CTAs per SM: 2 x (112 KB dynamic + 1 KB static + 1 KB per-block reservation) = 228 KB, exactly the H100's shared
// memory per SM, with no headroom.  The static part is the mbarriers padded to 1 KB by smem_raw's __align__(1024).  Any
// added static shared memory makes the occupancy check in y5obb_conv_create send every narrow layer back to one CTA
// (correct, but slower); y5obb_conv_schedule and tests/test_conv_schedule_gpu.py expose that.
constexpr int SMEM_PAIR = 112 * 1024;

// Epilogue staging per consumer warp, sized for the Detect head: 16 rows x min(NI, 64) fp32 columns, each row padded by 4
// (spreads the banks), then 16 theta indices.  A conv epilogue uses the first half of it: a 16 x min(NI, 64) bf16 output
// block, then a bf16 residual block of the same shape (see stg_chunk).
__host__ __device__ constexpr int stg_cols(int ni) { return ni < 64 ? ni : 64; }
__host__ __device__ constexpr int stg_pitch(int ni) { return stg_cols(ni) + 4; }
__host__ __device__ constexpr int stg_bytes(int ni) { return (16 * stg_pitch(ni) + 16) * 4; }
static_assert(2 * 16 * stg_cols(16) * 2 <= stg_bytes(16) && 2 * 16 * stg_cols(64) * 2 <= stg_bytes(64), "conv staging fits");

// Instantiations with NI <= 96 run two CTAs per SM: 2 x 384 threads at 80 registers each, of which setmaxnreg gives the
// producer warpgroup 32 and the consumers 104 (128 * 32 + 256 * 104 = 384 * 80).  Wider ones keep the SM to themselves,
// with 40 / 232 (up to 128 fp32 accumulators per consumer thread).
template <int NI>
struct Occupancy {
  static constexpr int CTAS = NI <= 96 ? 2 : 1;
  static constexpr int PRODUCER_REGS = CTAS == 2 ? 32 : 40;
  static constexpr int CONSUMER_REGS = CTAS == 2 ? 104 : 232;
};

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
  int det_descale;         // 1: test-time-augmentation branch, x y w h *= det_inv_scale, then x = det_flip_w - x if > 0
  float det_inv_scale, det_flip_w;
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

// fp16 plans (F16, Y5OBB_CONV_F16): cvt.rn.f16x2.f32 - overflow rounds to +-inf, as torch's half conversion does
__device__ __forceinline__ uint32_t pack_f16(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <bool F16>
__device__ __forceinline__ uint32_t pack_elem2(float a, float b) {
  if constexpr (F16) return pack_f16(a, b);
  else return pack_bf16(a, b);
}
template <bool F16>
__device__ __forceinline__ float2 unpack_elem2(uint32_t v) {
  if constexpr (F16) return __half22float2(*reinterpret_cast<const __half2*>(&v));
  else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
}
// the fp32 value of x rounded to fp16
__device__ __forceinline__ float r16(float x) { return __half2float(__float2half_rn(x)); }
// ATen's half sigmoid (fp32 opmath, IEEE division, one rounding to fp16) of the fp16 logit l
__device__ __forceinline__ float sigmoid16(float l) { return r16(__fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-l)))); }

__device__ __forceinline__ uint64_t desc_from(uint32_t lo, uint32_t hi) {
  uint64_t d;
  asm volatile("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}

// Y5OBB_DETECT_PROBE (tools/time_detect.py builds it into a library of its own): thread 0 of every CTA of a compact-record
// Detect launch stamps clock64 at each phase of its first PROBE_TILES tiles; y5obb_detect_probe copies the stamps out.
enum ProbePhase : int { PH_TILE = 0, PH_FULL, PH_MMA, PH_ARGMAX, PH_STAGED, PH_STORED, PROBE_PHASES };
#ifdef Y5OBB_DETECT_PROBE
constexpr int PROBE_CTAS = 264, PROBE_TILES = 64;
__device__ long long g_probe[PROBE_CTAS][PROBE_TILES][PROBE_PHASES];
__device__ __forceinline__ void probe(const ConvK& p, int ti, int ph) {
  if (p.mode == MODE_DETECT && p.det_decode == 2 && threadIdx.x == 0 && blockIdx.x < PROBE_CTAS && ti < PROBE_TILES)
    g_probe[blockIdx.x][ti][ph] = clock64();
}
#else
__device__ __forceinline__ void probe(const ConvK&, int, int) {}
#endif

// Y5OBB_CONV_PROBE (tools/time_conv_epilogue.py builds it into a library of its own): thread 0 of every CTA of a MODE_CONV
// launch adds the clock64 cycles since its previous stamp to the phase that each stamp ends, for its first CPROBE_TILES
// tiles.  The epilogue loops over 64-column blocks, so a phase is the SUM of its intervals within a tile.  CP_NEXT is the
// gap from the previous tile's last stamp to this tile's start.
enum ConvProbePhase : int { CP_NEXT = 0, CP_FULL, CP_MMA, CP_STAGED, CP_RES, CP_STORED, CONV_PROBE_PHASES };
#ifdef Y5OBB_CONV_PROBE
constexpr int CPROBE_CTAS = 264, CPROBE_TILES = 64;
__device__ long long g_cprobe[CPROBE_CTAS][CPROBE_TILES][CONV_PROBE_PHASES];
__device__ long long g_cprobe_last[CPROBE_CTAS];
__device__ __forceinline__ void cprobe(const ConvK& p, int ti, int ph) {
  if (p.mode == MODE_CONV && threadIdx.x == 0 && blockIdx.x < CPROBE_CTAS && ti < CPROBE_TILES) {
    const long long now = clock64();
    if (ti > 0 || ph != CP_NEXT) g_cprobe[blockIdx.x][ti][ph] += now - g_cprobe_last[blockIdx.x];
    g_cprobe_last[blockIdx.x] = now;
  }
}
// the same once `v` (a loaded value) has arrived: storing it makes the thread wait for the load
__device__ unsigned g_cprobe_sink;
__device__ __forceinline__ void cprobe_after(const ConvK& p, int ti, int ph, unsigned v) {
  if (threadIdx.x == 0) g_cprobe_sink = v;
  cprobe(p, ti, ph);
}
#else
__device__ __forceinline__ void cprobe(const ConvK&, int, int) {}
__device__ __forceinline__ void cprobe_after(const ConvK&, int, int, unsigned) {}
#endif

// ---- epilogue of one tile for one consumer warp ----------------------------------------------------------------------
// A 64-column block of a warp's 16 rows leaves as 16 * VECS 8-column vectors; lane `lane` stores vectors lane + 32 k, which
// are chunk lane % VECS of rows lane / VECS + k * ROW_STEP.
template <int NI>
struct StoreVecs {
  static constexpr int VECS = stg_cols(NI) / 8;     // 8-column vectors per staged row
  static constexpr int PER_LANE = 16 * VECS / 32;   // vectors per lane and block
  static constexpr int ROW_STEP = 32 / VECS;        // rows between a lane's vectors
  static constexpr int FRAG = stg_cols(NI) / 4;     // bf16 pairs per lane and block in the accumulator layout
  // blocks whose residual is loaded into registers (FRAG per lane) when the tile starts, so that the loads' latency passes
  // under the tile's MMAs: the first two for NI = 128, the first one otherwise (none for NI = 96, whose 48 accumulators
  // leave no room in the two-CTA budget; a second block spills at NI = 256); later blocks load in the epilogue.  DIM: the
  // array extent (at least 1).
  static constexpr int PREFETCH = NI == 96 ? 0 : (NI == 128 ? 2 : 1);
  static constexpr int DIM = PREFETCH > 0 ? PREFETCH : 1;
};

// residual vector k of this lane in the 64-column block at column cb, in the store layout (vector lane + 32 k); nullptr
// where the store loop stores nothing (columns past the tile or Cout, pixels past the image)
template <int NI>
__device__ __forceinline__ const __nv_bfloat16* res_vec(const ConvK& p, const TileCoord& c, int row0, int lane, int cb, int k) {
  constexpr int VECS = StoreVecs<NI>::VECS;
  const int v = lane + 32 * k;
  const int row = v / VECS, col = cb + (v % VECS) * 8;
  const int tr = row0 + row;
  const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
  const int h = c.h0 + hl, w = c.w0 + (tr - hl * p.Wt);
  if (col >= min(p.BN, p.Cout - c.n0) || h >= p.Hout || w >= p.Wout) return nullptr;
  return p.res + (long long)c.b * p.res_img_stride + (long long)h * p.res_row_stride + (long long)w * p.res_pix_stride + c.n0 +
         col;
}
// the residual of the 64-column block at column cb in the accumulator layout: rf[2 jj + i] holds row row0 + lane / 4 + 8 i,
// columns cb + 8 jj + 2 (lane % 4) (+ 1) as bf16x2 (4-byte loads; a quad reads 16 contiguous bytes of a pixel); zero where
// nothing is stored
template <int NI>
__device__ __forceinline__ void load_res_frag(const ConvK& p, const TileCoord& c, int row0, int lane, int cb,
                                              uint32_t (&rf)[StoreVecs<NI>::FRAG]) {
  const int nvalid = min(p.BN, p.Cout - c.n0), col = cb + 2 * (lane & 3);
  const __nv_bfloat16* rp[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int tr = row0 + (lane >> 2) + 8 * i;
    const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
    const int h = c.h0 + hl, w = c.w0 + (tr - hl * p.Wt);
    rp[i] = h < p.Hout && w < p.Wout
                ? p.res + (long long)c.b * p.res_img_stride + (long long)h * p.res_row_stride + (long long)w * p.res_pix_stride +
                      c.n0 + col
                : nullptr;
  }
#pragma unroll
  for (int jj = 0; jj < StoreVecs<NI>::FRAG / 2; ++jj)
#pragma unroll
    for (int i = 0; i < 2; ++i)
      rf[2 * jj + i] = rp[i] && col + 8 * jj < nvalid ? *reinterpret_cast<const uint32_t*>(rp[i] + 8 * jj) : 0u;
}

// Byte offset of 16-byte chunk i (row i / VECS, 8-column group i % VECS) of a conv staging block.  The chunks of each
// 128-byte line are permuted by XOR with the line's index, so that the eight rows of one column group (an stmatrix /
// ldmatrix matrix) and eight consecutive chunks (a quarter-warp of the store loop) fall in eight different bank quads.
__device__ __forceinline__ uint32_t stg_chunk(uint32_t i) { return (i ^ ((i >> 3) & 7u)) << 4; }

// MODE_CONV.  The warp owns 16 pixel rows (row0 .. row0 + 15 of the tile).  wgmma's accumulator layout gives thread
// `lane` the rows row0 + lane / 4 (+ 8) and the column pairs 8 j + 2 (lane % 4) (+ 1): for each pair of 8-column groups,
// exactly the four 8 x 8 matrices of one stmatrix.x4.  Per 64-column block: bias (+ SiLU) in registers, the residual
// (RES) added in fp32 in registers, one rounding to bf16 (fp16 when F16), the block staged as [16 rows][64] bf16 by stmatrix, and 16-byte
// stores per pixel.  RES: rpf holds the residual of the first StoreVecs<NI>::PREFETCH blocks in the accumulator layout,
// loaded when the tile started; a later block's residual is copied by cp.async into the staging area's second half in the
// store layout and comes back in the accumulator layout by ldmatrix.  The probe's phases: CP_STAGED the activation and
// the staging, CP_RES the wait for the residual, CP_STORED the stores.
template <int NI, bool RES, bool F16>
__device__ __forceinline__ void epilogue(const ConvK& p, const TileCoord& c, float (&acc)[NI / 2], float* stg, const float* bias_s,
                                         const uint32_t (&rpf)[StoreVecs<NI>::DIM][StoreVecs<NI>::FRAG], int row0,
                                         int lane, int ti) {
  constexpr int VECS = StoreVecs<NI>::VECS, PER_LANE = StoreVecs<NI>::PER_LANE, ROW_STEP = StoreVecs<NI>::ROW_STEP;
  const int q = lane & 3;
  const int nvalid = min(p.BN, p.Cout - c.n0);
  const float* bias = bias_s + c.n0;
  const uint32_t out_s = ptx::smem_u32(stg), res_s = out_s + 16 * stg_cols(NI) * 2;
  // stmatrix / ldmatrix: lane gives the address of row lane % 16 of column group 2 jp + lane / 16
  const uint32_t mat = (uint32_t)((lane & 15) * VECS + (lane >> 4));
  // The store loop's vectors of this lane: column vcol of rows lane / VECS + k * ROW_STEP, whose pixels are found once per
  // tile: hw[k] = (hl << 16) | wl, the pixel's row and column within the tile (-1 past the image), from obase / obase2x.
  const int vcol = (lane % VECS) * 8;
  int hw[PER_LANE];
  __nv_bfloat16* obase;
  __nv_bfloat16* obase2x;
#pragma unroll
  for (int cb = 0; cb < NI; cb += 64) {
    if (cb >= nvalid) break;
    const bool prefetched = cb / 64 < StoreVecs<NI>::PREFETCH;
    if constexpr (RES) {  // a later block's residual is copied here, straight into shared memory, and lands while (1) runs
      if (!prefetched) {
#pragma unroll
        for (int k = 0; k < PER_LANE; ++k) {
          const __nv_bfloat16* src = res_vec<NI>(p, c, row0, lane, cb, k);
          ptx::cp_async_16(res_s + stg_chunk(lane + 32 * k), src ? src : p.res, src ? 16u : 0u);
        }
      }
    }
    // (1) bias (+ SiLU) in registers, in place
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int j = cb / 8 + jj;
      if (j < NI / 8) {
        const int col = 8 * j + 2 * q;
        const float b0 = bias[col], b1 = bias[col + 1];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float& v0 = acc[4 * j + 2 * i];
          float& v1 = acc[4 * j + 2 * i + 1];
          if (p.act) {  // SiLU(x) = h + h * tanh(h), h = x / 2 = 0.5 * acc + (0.5 * bias)
            const float h0 = fmaf(v0, 0.5f, b0), h1 = fmaf(v1, 0.5f, b1);
            v0 = fmaf(h0, tanh_fast(h0), h0);
            v1 = fmaf(h1, tanh_fast(h1), h1);
          } else {
            v0 += b0;
            v1 += b1;
          }
        }
      }
    }
    cprobe(p, ti, CP_STAGED);
    if constexpr (RES) {
      if (prefetched) {
        cprobe_after(p, ti, CP_RES, rpf[cb / 64][0] ^ rpf[cb / 64][StoreVecs<NI>::FRAG - 1]);
      } else {
        ptx::cp_async_wait_all();
        cprobe(p, ti, CP_RES);
        __syncwarp();
      }
    }
    // (2) (+ residual in fp32), one rounding to bf16, staged by stmatrix: matrix m of column-group pair jp is group
    // 2 jp + m / 2, rows 8 (m % 2) .. 8 (m % 2) + 7
#pragma unroll
    for (int jp = 0; jp < 4; ++jp) {
      const int j0 = cb / 8 + 2 * jp;
      if (j0 < NI / 8 && 2 * jp < VECS) {
        uint32_t rb[4];
        if constexpr (RES) {
          if (prefetched) {  // (the index stays in range in the unrolled blocks where this branch is dead)
#pragma unroll
            for (int m = 0; m < 4; ++m) rb[m] = rpf[prefetched ? cb / 64 : 0][4 * jp + m];
          } else {
            ptx::ldmatrix_x4(res_s + stg_chunk(mat + 2 * jp), rb);
          }
        }
        uint32_t o[4];
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          float f0 = acc[4 * (j0 + m / 2) + 2 * (m % 2)], f1 = acc[4 * (j0 + m / 2) + 2 * (m % 2) + 1];
          if constexpr (RES) {
            const float2 g = unpack_elem2<F16>(rb[m]);
            f0 += g.x;
            f1 += g.y;
          }
          o[m] = pack_elem2<F16>(f0, f1);
        }
        ptx::stmatrix_x4(out_s + stg_chunk(mat + 2 * jp), o);
      }
    }
    __syncwarp();
    cprobe(p, ti, CP_STAGED);
    if (cb == 0) {  // once per tile, after the first block's accumulators are staged (fewer registers live)
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) {
        const int tr = row0 + lane / VECS + k * ROW_STEP;
        const int hl = (int)fdiv((uint32_t)tr, p.fd_wt), wl = tr - hl * p.Wt;
        hw[k] = c.h0 + hl < p.Hout && c.w0 + wl < p.Wout ? (hl << 16) | wl : -1;
      }
      obase = p.out + (long long)c.b * p.out_img_stride + (long long)c.h0 * p.out_row_stride + (long long)c.w0 * p.out_pix_stride +
              c.n0 + vcol;
      obase2x = p.out2x ? p.out2x + (((long long)c.b * 2 * p.Hout + 2 * c.h0) * (2 * p.Wout) + 2 * c.w0) * p.out2x_pix_stride +
                              c.n0 + vcol
                        : nullptr;
    }
    // (3) 16 rows x (up to) 64 columns leave in vectors
    if (cb + vcol < nvalid) {
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) {
        if (hw[k] < 0) continue;
        const int hl = hw[k] >> 16, wl = hw[k] & 0xFFFF;
        const uint4 o = ptx::ld_shared_u4(out_s + stg_chunk(lane + 32 * k));
        *reinterpret_cast<uint4*>(obase + hl * p.out_row_stride + wl * p.out_pix_stride + cb) = o;
        if (obase2x) {  // nn.Upsample(2x nearest): the same vector on the four (dy, dx) phases
          const long long px = p.out2x_pix_stride, rw = 2LL * p.Wout * px;
          __nv_bfloat16* u = obase2x + (2 * hl * rw + 2 * wl * px) + cb;
          *reinterpret_cast<uint4*>(u) = o;
          *reinterpret_cast<uint4*>(u + px) = o;
          *reinterpret_cast<uint4*>(u + rw) = o;
          *reinterpret_cast<uint4*>(u + rw + px) = o;
        }
      }
    }
    cprobe(p, ti, CP_STORED);
    __syncwarp();
  }
}

// F16 decode of the first four columns (f: their fp16 sigmoids) of anchor a at grid cell (gx, gy), as models/yolo.py:72-73
// computes it on a half y: xy = fp16((fp16(2 y - 0.5) + grid) * stride), wh = fp16(fp16((2 y)^2) * anchor_grid), and
// _descale_pred's half `/= s` (a multiply by the fp32 1/s) and `W - x`.  2 y, 2 y - 0.5 and (2 y)^2 are exact in fp32.
__device__ __forceinline__ void decode16(const ConvK& p, float (&f)[4], float gx, float gy, int a) {
  f[0] = r16(__fmul_rn(__fadd_rn(r16(__fsub_rn(2.0f * f[0], 0.5f)), gx), p.det_stride));
  f[1] = r16(__fmul_rn(__fadd_rn(r16(__fsub_rn(2.0f * f[1], 0.5f)), gy), p.det_stride));
  f[2] = r16(__fmul_rn(r16(__fmul_rn(2.0f * f[2], 2.0f * f[2])), p.det_anchor[2 * a]));
  f[3] = r16(__fmul_rn(r16(__fmul_rn(2.0f * f[3], 2.0f * f[3])), p.det_anchor[2 * a + 1]));
  if (p.det_descale) {
#pragma unroll
    for (int k = 0; k < 4; ++k) f[k] = r16(__fmul_rn(f[k], p.det_inv_scale));
    if (p.det_flip_w > 0.0f) f[0] = r16(__fsub_rn(p.det_flip_w, f[0]));
  }
}

// MODE_DETECT through the shared epilogue (every Detect launch that is not epilogue_records').  Each 64-column block is
// activated in registers, staged through shared memory as [16 rows][64] fp32 and leaves as fp32 rows.
// F16: models/yolo.py:63-77 on a half tensor, operation by operation.  Each logit is rounded to fp16 (the conv's output),
// sigmoid16 activates it, the decode rounds to fp16 where torch stores a half tensor (grid, stride and anchor_grid are
// fp32, so their add and multiplies run in fp32 first), the theta index is the first maximum of the 180 fp16 sigmoids,
// and rows other than records leave as fp16.
template <int NI, bool F16>
__device__ __forceinline__ void epilogue_detect(const ConvK& p, const TileCoord& c, float (&acc)[NI / 2], float* stg,
                                                const float* bias_s, int row0, int lane, int ti) {
  const int q = lane & 3, r = lane >> 2;
  constexpr int PITCH = stg_pitch(NI);
  float* theta_s = stg + 16 * PITCH;
  const int nfix = p.det_no - 180;  // 5 + nc leading columns, then the theta bins
  const float* bias = bias_s + c.n0;
  if (p.det_decode == 2) {
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
            float v = acc[4 * j + 2 * i + k] + bias[col];
            if constexpr (F16) v = sigmoid16(r16(v));
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
    probe(p, ti, PH_ARGMAX);
  }
  const int ncols = p.det_decode == 2 ? p.det_rec_w : min(p.BN, p.det_no);  // columns that leave the kernel
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
          if constexpr (F16) {
            v0 = r16(v0);
            v1 = r16(v1);
          }
          *reinterpret_cast<float2*>(stg + (r + 8 * i) * PITCH + (col - cb)) = make_float2(v0, v1);
        }
      }
    }
    __syncwarp();
    probe(p, ti, PH_STAGED);
    // (2) Detect, N tile nt == anchor nt.  Output row = b * rows_per_image + row_off + (a * H + h) * W + w (models/yolo.py):
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
      const float4 x = *reinterpret_cast<const float4*>(stg + row * PITCH + (col - cb));
      float f[4] = {x.x, x.y, x.z, x.w};
      if (p.det_decode) {
#pragma unroll
        for (int k = 0; k < 4; ++k) f[k] = F16 ? sigmoid16(f[k]) : sigmoid_fast(f[k]);
        if (F16 && col == 0) {
          decode16(p, f, (float)w, (float)h, a);
        } else if (col == 0) {  // xy, wh (models/yolo.py)
          f[0] = (f[0] * 2.0f - 0.5f + (float)w) * p.det_stride;
          f[1] = (f[1] * 2.0f - 0.5f + (float)h) * p.det_stride;
          f[2] = (f[2] * 2.0f) * (f[2] * 2.0f) * p.det_anchor[2 * a];
          f[3] = (f[3] * 2.0f) * (f[3] * 2.0f) * p.det_anchor[2 * a + 1];
          if (p.det_descale) {  // _descale_pred (models/yolo.py:183-198): ATen's `/= s` is a multiply by the fp32 1/s,
                                // the lr de-flip W - x; _rn so that neither contracts into the decode's FMAs
#pragma unroll
            for (int k = 0; k < 4; ++k) f[k] = __fmul_rn(f[k], p.det_inv_scale);
            if (p.det_flip_w > 0.0f) f[0] = __fsub_rn(p.det_flip_w, f[0]);
          }
        }
        if (p.det_decode == 2) {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (col + k >= nfix) f[k] = col + k == nfix ? theta_s[row] : 0.0f;
        }
      }
      const long long orow = (long long)c.b * p.det_rows_per_image + p.det_row_off + ((long long)a * p.Hout + h) * p.Wout + w;
      if (F16 && p.det_decode != 2) {  // fp16 rows: 8-byte vectors when rows are 4-aligned, element stores otherwise
        __half* dst = reinterpret_cast<__half*>(p.det_out) + orow * rw + col;
        if (!(rw & 3)) {
          *reinterpret_cast<uint2*>(dst) = make_uint2(pack_f16(f[0], f[1]), pack_f16(f[2], f[3]));
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (col + k < ncols) dst[k] = __float2half_rn(f[k]);
        }
        continue;
      }
      float* dst = p.det_out + orow * rw + col;
      if (!(rw & 3)) {
        *reinterpret_cast<float4*>(dst) = make_float4(f[0], f[1], f[2], f[3]);
      } else {  // det_no % 4 != 0 (records are always 4-aligned): rows start 4-byte aligned and the last vector ends the row early
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (col + k < ncols) dst[k] = f[k];
      }
    }
    __syncwarp();
  }
  probe(p, ti, PH_STORED);
}

// ---- compact-record Detect epilogue (det_decode 2, det_rec_w <= 64) -----------------------------------------------------
// The same record, bit for bit, as epilogue<NI>'s records branch: the same fp32 expressions on the same accumulators, only
// scheduled differently.  Thread `lane` holds rows row0 + r (+ 8) and columns 8 j + 2 q (+ 1), q = lane % 4, r = lane / 4.
//
// bt_s, NI floats behind the bias in shared memory, holds the CTA's current anchor's theta biases: bias[col] for the 180
// theta bins (nfix <= col < det_no), -inf for every other column.  acc + (-inf) is -inf, or NaN for an infinite acc, and
// neither is ever > best, so the arg-max needs no column test: it is straight-line load / add / compare / select code.
// (Registers would be faster still, but the accumulators already take 112 of the 168 that ptxas may allocate.)
//
// The record (cx, cy, w, h, obj, cls[nc], theta index, zero padding) of each row is built in registers and written once to
// the warp's staging buffer as [16 rows][det_rec_w] fp32 - the layout of 16 consecutive output rows.  Rows that are
// consecutive pixels of one image row (all 16 when the tile spans whole image rows, Wt == Wout) are consecutive records of
// [B, A, rec_w], so each run of them leaves in one cp.async.bulk store.  The store reads the staging buffer asynchronously;
// the next tile's epilogue waits for that read before it writes the buffer again, so the store overlaps the next tile's MMAs.
// F16: the record of epilogue_detect<NI, true> - fp16 logits, sigmoid16, decode16, and the first maximum of the 180 fp16
// sigmoids, which rounding can tie where the logits differ.  The -inf of a non-theta column stays -inf instead.
template <int NI, bool F16>
__device__ __forceinline__ void epilogue_records(const ConvK& p, const TileCoord& c, float (&acc)[NI / 2], const float* bt_s,
                                                 float* stg, const float* bias_s, int row0, int lane, int ti) {
  const int q = lane & 3, r = lane >> 2;
  const int nfix = p.det_no - 180, rw = p.det_rec_w;
  // (1) theta: the first maximum of acc + bias over the 180 bins.  Per thread in increasing column order (strict >), then
  // across the quad (larger value, or equal value and smaller column) - epilogue<NI>'s order and tie rule.  bk holds the
  // column; nfix (bin 0) is what a row without any finite logit reports, as there.
  float best[2] = {-INFINITY, -INFINITY};
  int bk[2] = {nfix, nfix};
  const uint32_t bt_u = ptx::smem_u32(bt_s + 2 * q);
#pragma unroll
  for (int j = 0; j < NI / 8; ++j) {
    const float2 bt = ptx::ld_shared_v2(bt_u + 32u * j);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float b = k ? bt.y : bt.x;
        float v = acc[4 * j + 2 * i + k] + b;
        if constexpr (F16) v = b == -INFINITY ? -INFINITY : sigmoid16(r16(v));
        const bool take = v > best[i];
        best[i] = take ? v : best[i];
        bk[i] = take ? 8 * j + 2 * q + k : bk[i];
      }
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best[i], off);
      const int ok = __shfl_xor_sync(0xffffffffu, bk[i], off);
      const bool take = ob > best[i] || (ob == best[i] && ok < bk[i]);
      best[i] = take ? ob : best[i];
      bk[i] = take ? ok : bk[i];
    }
  probe(p, ti, PH_ARGMAX);

  // (2) sigmoid and decode in registers, straight into the staged records
  const int a = c.nt;
  float px[2], py[2];  // the grid cell (w, h) of the thread's two rows
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int tr = row0 + r + 8 * i;
    const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
    px[i] = (float)(c.w0 + (tr - hl * p.Wt));
    py[i] = (float)(c.h0 + hl);
  }
  const float* bias = bias_s + c.n0;
  const uint32_t stg_u = ptx::smem_u32(stg);
  ptx::tma_store_wait_read<0>();  // the previous tile's bulk stores have read the staging buffer
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 8; ++j) {  // det_rec_w <= 64
    const int col = 8 * j + 2 * q;
    if (8 * j >= rw) break;
    if (col >= rw) continue;
    const float2 b = col < nfix ? ptx::ld_shared_v2(ptx::smem_u32(bias + col)) : make_float2(0.0f, 0.0f);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float f0, f1;
      if constexpr (F16) {
        f0 = sigmoid16(r16(acc[4 * j + 2 * i] + b.x));
        f1 = sigmoid16(r16(acc[4 * j + 2 * i + 1] + b.y));
      } else {
        f0 = sigmoid_fast(acc[4 * j + 2 * i] + b.x);
        f1 = sigmoid_fast(acc[4 * j + 2 * i + 1] + b.y);
      }
      if (F16 && j == 0 && q < 2) {  // decode16's columns 0, 1 (q = 0) or 2, 3 (q = 1)
        float f[4] = {f0, f1, f0, f1};
        decode16(p, f, px[i], py[i], a);
        f0 = q == 0 ? f[0] : f[2];
        f1 = q == 0 ? f[1] : f[3];
      } else if (j == 0 && q < 2) {  // xy, wh (models/yolo.py)
        if (q == 0) {
          f0 = (f0 * 2.0f - 0.5f + px[i]) * p.det_stride;
          f1 = (f1 * 2.0f - 0.5f + py[i]) * p.det_stride;
        } else {
          f0 = (f0 * 2.0f) * (f0 * 2.0f) * p.det_anchor[2 * a];
          f1 = (f1 * 2.0f) * (f1 * 2.0f) * p.det_anchor[2 * a + 1];
        }
        if (p.det_descale) {  // _descale_pred, as in epilogue<NI>
          f0 = __fmul_rn(f0, p.det_inv_scale);
          f1 = __fmul_rn(f1, p.det_inv_scale);
          if (q == 0 && p.det_flip_w > 0.0f) f0 = __fsub_rn(p.det_flip_w, f0);
        }
      }
      const float th = (float)(bk[i] - nfix);
      if (col >= nfix) f0 = col == nfix ? th : 0.0f;
      if (col + 1 >= nfix) f1 = col + 1 == nfix ? th : 0.0f;
      ptx::st_shared_v2(stg_u + (uint32_t)(((r + 8 * i) * rw + col) * 4), f0, f1);
    }
  }
  ptx::fence_proxy_async();  // the staged records, written through the generic proxy, are read by the bulk copy
  __syncwarp();
  probe(p, ti, PH_STAGED);

  // (3) lane l < 16 describes row l: its output row, and whether a run of consecutive output rows starts there
  const int l = lane & 15;
  const int tr = row0 + l;
  const int hl = (int)fdiv((uint32_t)tr, p.fd_wt);
  const int h = c.h0 + hl, w = c.w0 + (tr - hl * p.Wt);
  const bool valid = lane < 16 && h < p.Hout && w < p.Wout;
  const long long orow = (long long)c.b * p.det_rows_per_image + p.det_row_off + ((long long)a * p.Hout + h) * p.Wout + w;
  const long long prev = __shfl_up_sync(0xffffffffu, orow, 1);
  const uint32_t vmask = __ballot_sync(0xffffffffu, valid);
  const bool start = valid && (l == 0 || !((vmask >> (l - 1)) & 1u) || prev + 1 != orow);
  const uint32_t smask = __ballot_sync(0xffffffffu, start);
  if (start) {
    const uint32_t brk = ((smask | ~vmask) & (0xFFFFFFFEu << l)) | (1u << 16);  // the first row after l that ends the run
    const int len = __ffs(brk) - 1 - l;
    ptx::bulk_store(p.det_out + orow * rw, stg + l * rw, (uint32_t)(len * rw * 4));
    ptx::tma_store_commit();
  }
  probe(p, ti, PH_STORED);
}

// RECORDS: the Detect head with compact records (epilogue_records); otherwise epilogue_detect for the other Detect launches
// and epilogue<NI, RES> for every conv.  RES: a MODE_CONV launch with a residual, whose residual vectors are loaded when
// each tile starts.
template <int NI, bool RECORDS, bool RES = false, bool F16 = false>
__global__ void __launch_bounds__(NUM_THREADS, Occupancy<NI>::CTAS) conv_wgmma_kernel(const __grid_constant__ ConvK p) {
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
  float* bias_s = reinterpret_cast<float*>(stg_all + (size_t)CONSUMER_WARPS * stg_bytes(NI));

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
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(Occupancy<NI>::PRODUCER_REGS));
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
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(Occupancy<NI>::CONSUMER_REGS));
  for (int i = threadIdx.x; i < p.cout_pad + 32; i += 32 * CONSUMER_WARPS) bias_s[i] = __ldg(p.bias + i);
  asm volatile("bar.sync 1, %0;" ::"n"(32 * CONSUMER_WARPS) : "memory");
  if (p.b_resident) ptx::mbar_wait(&wres_bar, 0u);

  const int wg = warp >> 2;
  float* stg = reinterpret_cast<float*>(stg_all + (size_t)warp * stg_bytes(NI));
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
  float* bt_s = bias_s + ((p.cout_pad + 32 + 31) & ~31);  // epilogue_records: the theta biases of anchor bt_nt
  int bt_nt = -1;
  int s = 0, prev_s = -1, ti = 0;
  uint32_t ph = 0, s_lo = ring_lo;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x, ++ti) {
    const TileCoord c = decode_tile(p, t);
    uint32_t scale_d = 0u, bres_lo = res_lo;
    int kc = 0;
    probe(p, ti, PH_TILE);
    cprobe(p, ti, CP_NEXT);
    uint32_t rpf[StoreVecs<NI>::DIM][StoreVecs<NI>::FRAG];  // RES: residual fragments, in flight under the MMAs
    if constexpr (RES) {
#pragma unroll
      for (int b = 0; b < StoreVecs<NI>::PREFETCH; ++b) load_res_frag<NI>(p, c, wg * 64 + (warp & 3) * 16, lane, 64 * b, rpf[b]);
    }
    for (int u0 = 0; u0 < n_units; u0 += group) {
      const int ng = min(group, n_units - u0);
      ptx::mbar_wait(&full_bar[s], ph);
      if (u0 == 0) {
        probe(p, ti, PH_FULL);
        cprobe(p, ti, CP_FULL);
      }
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
            ptx::Wgmma<NI>::template mma<0, 0, F16>(acc, desc_from(a_lo + (uint32_t)u * a_step + 2u * j, hi),
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
    probe(p, ti, PH_MMA);
    cprobe(p, ti, CP_MMA);
    if constexpr (RECORDS) {
      if (c.nt != bt_nt) {  // every consumer warp walks the same tiles, so all of them come here together
        asm volatile("bar.sync 1, %0;" ::"n"(32 * CONSUMER_WARPS) : "memory");  // no warp reads the old anchor's any more
        const int nfix = p.det_no - 180;
        for (int col = threadIdx.x; col < NI; col += 32 * CONSUMER_WARPS)
          bt_s[col] = (col >= nfix && col < p.det_no) ? bias_s[c.n0 + col] : -INFINITY;
        asm volatile("bar.sync 1, %0;" ::"n"(32 * CONSUMER_WARPS) : "memory");
        bt_nt = c.nt;
      }
      epilogue_records<NI, F16>(p, c, acc, bt_s, stg, bias_s, wg * 64 + (warp & 3) * 16, lane, ti);
    } else if (p.mode == MODE_DETECT) {
      if constexpr (!RES) epilogue_detect<NI, F16>(p, c, acc, stg, bias_s, wg * 64 + (warp & 3) * 16, lane, ti);
    } else {
      epilogue<NI, RES, F16>(p, c, acc, stg, bias_s, rpf, wg * 64 + (warp & 3) * 16, lane, ti);
    }
  }
  if constexpr (RECORDS) ptx::tma_store_wait_all();  // the records' bulk stores complete before the CTA exits
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
int ctas_for(int ni) { return ni <= 96 ? 2 : 1; }  // Occupancy<NI>::CTAS
template <bool RES, bool F16>
KernelFn kernel_for(int ni) {
  switch (ni) {
    case 16: return conv_wgmma_kernel<16, false, RES, F16>;
    case 32: return conv_wgmma_kernel<32, false, RES, F16>;
    case 64: return conv_wgmma_kernel<64, false, RES, F16>;
    case 96: return conv_wgmma_kernel<96, false, RES, F16>;
    case 128: return conv_wgmma_kernel<128, false, RES, F16>;
    case 160: return conv_wgmma_kernel<160, false, RES, F16>;
    case 192: return conv_wgmma_kernel<192, false, RES, F16>;
    case 224: return conv_wgmma_kernel<224, false, RES, F16>;
    case 256: return conv_wgmma_kernel<256, false, RES, F16>;
    default: return nullptr;
  }
}
// compact records need det_no > 180, so an N tile of at least 192 columns
template <bool F16>
KernelFn records_kernel_for(int ni) {
  switch (ni) {
    case 192: return conv_wgmma_kernel<192, true, false, F16>;
    case 224: return conv_wgmma_kernel<224, true, false, F16>;
    case 256: return conv_wgmma_kernel<256, true, false, F16>;
    default: return nullptr;
  }
}

struct ConvObj {
  ConvK k;
  KernelFn fn;
  int grid;
  int ctas_per_sm;   // 1, or 2 for the NI <= 96 instantiations when their plan fits half of the shared memory
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
  // compact records take epilogue_records when a record fits the 64-column staging row (nc <= 58)
  const bool records = d->mode == MODE_DETECT && d->det_decode == 2 && d->det_no > 180 &&
                       ((d->det_no - 180 + 1) + 3) / 4 * 4 <= 64 && !(d->flags & Y5OBB_CONV_DETECT_GENERIC);
  const bool res_epi = d->mode == MODE_CONV && d->res;  // residual vectors loaded when each tile starts
  const bool f16 = (d->flags & Y5OBB_CONV_F16) != 0;
  if (f16)
    o->fn = records ? records_kernel_for<true>(ni) : (res_epi ? kernel_for<true, true>(ni) : kernel_for<false, true>(ni));
  else
    o->fn = records ? records_kernel_for<false>(ni) : (res_epi ? kernel_for<true, false>(ni) : kernel_for<false, false>(ni));
  const int inst = (records ? 1 : (res_epi ? 2 : 0)) + (f16 ? 3 : 0);
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
  // the bias lives in shared memory behind the staging buffers (records: then NI floats of theta biases, see bt_s)
  const size_t bias_bytes = align_up((size_t)(cout_pad + 32) * 4, 128) + (records ? (size_t)ni * 4 : 0);
  const size_t fixed_bytes = 1024 + (size_t)CONSUMER_WARPS * stg_bytes(ni) + bias_bytes;  // alignment slack, staging, bias
  size_t SMEM_BUDGET = 0;  // for the operand ring and the resident weights: set per CTAs-per-SM choice below
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
  // Row shift sums the (tap, K-chunk) terms in another order than one load per tap.  That order is fixed here, by the
  // full-SM plan with 64-column staging, and every plan below keeps it: the schedule never changes a result bit.
  SMEM_BUDGET = (size_t)SMEM_TOTAL - (1024 + (size_t)CONSUMER_WARPS * stg_bytes(64) + bias_bytes);
  const bool rowshift_order = want_rowshift && plan(true);
  // Narrow instantiations share the SM between two CTAs when the layer's plan fits half of the shared memory: while one
  // CTA runs a tile's epilogue (or waits on its residual loads) the other's MMAs and loads go on.
  auto plan_for = [&](int ctas) -> bool {
    const size_t cap = ctas == 2 ? (size_t)SMEM_PAIR : (size_t)SMEM_TOTAL;
    if (cap <= fixed_bytes) return false;
    SMEM_BUDGET = cap - fixed_bytes;
    return plan(rowshift_order);
  };
  o->ctas_per_sm = 1;
  if (ctas_for(ni) == 2 && !(d->flags & Y5OBB_CONV_ONE_CTA) && plan_for(2)) o->ctas_per_sm = 2;
  if (o->ctas_per_sm == 1 && !plan_for(1)) {
    delete o;
    return Y5OBB_EINVAL;
  }
  static bool attr_set[6][257] = {};  // per instantiation (NI; plain, records, residual; bf16, then fp16)
  if (!attr_set[inst][ni]) {
    // all of the unified L1 / shared memory as shared memory, so that two 112 KB CTAs fit beside each other
    cudaError_t e = cudaFuncSetAttribute(o->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL);
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(o->fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) {
      delete o;
      return cuda_fail(e);
    }
    attr_set[inst][ni] = true;
  }
  auto smem_of_plan = [&]() { return k.b_res_bytes + (size_t)k.stages * stage_bytes + fixed_bytes; };
  o->smem = smem_of_plan();
  if (o->ctas_per_sm == 2) {  // the occupancy calculator has the last word; a plan that would run alone takes the full-SM plan
    int blocks = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, o->fn, NUM_THREADS, o->smem);
    if (e != cudaSuccess) {
      delete o;
      return cuda_fail(e);
    }
    if (blocks < 2) {
      o->ctas_per_sm = 1;
      if (!plan_for(1)) {
        delete o;
        return Y5OBB_EINVAL;
      }
      o->smem = smem_of_plan();
    }
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
  k.det_descale = d->det_descale ? 1 : 0;
  k.det_inv_scale = d->det_inv_scale;
  k.det_flip_w = d->det_flip_w;
  if (d->det_descale && (d->mode != MODE_DETECT || !d->det_decode || !(d->det_inv_scale > 0.0f) || d->det_flip_w < 0.0f)) {
    delete o;
    return Y5OBB_EINVAL;
  }
  if (d->mode == MODE_CONV) {
    if (!d->out || d->out_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->out) & 15) || d->Cout % 8 ||
        (d->res && (d->res_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->res) & 15))) ||
        (d->out2x && (d->out2x_pix_stride % 8 || (reinterpret_cast<uintptr_t>(d->out2x) & 15)))) {
      delete o;
      return Y5OBB_EINVAL;
    }
  } else {
    // rows of rw floats: 16-byte vector stores when rw % 4 == 0 (always for records), element stores otherwise
    // (fp16 plans write fp16 rows, 8-byte vectors, unless they write records)
    const int rw = d->det_decode == 2 ? k.det_rec_w : d->det_no;
    const bool half_rows = f16 && d->det_decode != 2;
    const uintptr_t align = half_rows ? (rw % 4 ? 1 : 7) : (rw % 4 ? 3 : 15);
    if (!d->det_out || (d->det_decode == 2 && d->det_no <= 180) ||
        ((reinterpret_cast<uintptr_t>(d->det_out) + (size_t)d->det_row_off * rw * (half_rows ? 2 : 4)) & align)) {
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
    CUresult r = enc(&k.tmA, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(d->in), dims, strides, box, es,
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
    CUresult r = enc(&k.tmB, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(d->w), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for(bk), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      g_last_cuda_error = (int)r;
      delete o;
      return Y5OBB_ECUDA;
    }
  }
  const int total = k.n_tiles_m * k.n_tiles_n;
  o->grid = std::min(total, o->ctas_per_sm * sm_count());
  if (k.b_resident && k.n_tiles_n > 1) o->grid = o->grid / k.n_tiles_n * k.n_tiles_n;  // one N tile per CTA (resident weights)
  o->threads = NUM_THREADS;
  o->flops = 2.0 * d->B * Hout * Wout * (double)d->Cout * d->Cin * d->KH * d->KW;
  o->hbm_bytes = 2.0 * d->B * ((double)d->Hin * d->Win * (d->hbm_cin ? d->hbm_cin : d->Cin) + (double)Hout * Wout * d->Cout * (d->res ? 2 : 1));
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

int y5obb_conv_schedule(const y5obb_conv_t* conv, int* ctas_per_sm, int* resident, int* rowshift, int* group) {
  if (!conv) return Y5OBB_EINVAL;
  const ConvObj* o = reinterpret_cast<const ConvObj*>(conv);
  if (ctas_per_sm) *ctas_per_sm = o->ctas_per_sm;
  if (resident) *resident = o->k.b_resident;
  if (rowshift) *rowshift = o->k.rowshift;
  if (group) *group = o->k.group;
  return Y5OBB_OK;
}

void y5obb_conv_destroy(y5obb_conv_t* conv) { delete reinterpret_cast<ConvObj*>(conv); }

}  // extern "C"

#ifdef Y5OBB_DETECT_PROBE
// the probe build's stamps (see g_probe): copies them to `host` ([PROBE_CTAS][PROBE_TILES][PROBE_PHASES] int64, `bytes` long)
// and zeroes them; returns the element count of each dimension in dims[3]
extern "C" int y5obb_detect_probe(void* host, size_t bytes, int* dims) {
  if (bytes < sizeof(g_probe) || !host || !dims) return Y5OBB_EINVAL;
  cudaError_t e = cudaMemcpyFromSymbol(host, g_probe, sizeof(g_probe));
  static long long zeros[PROBE_CTAS][PROBE_TILES][PROBE_PHASES];
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_probe, zeros, sizeof(g_probe));
  if (e != cudaSuccess) return cuda_fail(e);
  dims[0] = PROBE_CTAS;
  dims[1] = PROBE_TILES;
  dims[2] = PROBE_PHASES;
  return Y5OBB_OK;
}
#endif

#ifdef Y5OBB_CONV_PROBE
// the conv probe build's per-phase cycle sums (see g_cprobe): copies them to `host` ([CPROBE_CTAS][CPROBE_TILES]
// [CONV_PROBE_PHASES] int64, `bytes` long) and zeroes them; returns the element count of each dimension in dims[3]
extern "C" int y5obb_conv_probe(void* host, size_t bytes, int* dims) {
  if (bytes < sizeof(g_cprobe) || !host || !dims) return Y5OBB_EINVAL;
  cudaError_t e = cudaMemcpyFromSymbol(host, g_cprobe, sizeof(g_cprobe));
  static long long zeros[CPROBE_CTAS][CPROBE_TILES][CONV_PROBE_PHASES];
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_cprobe, zeros, sizeof(g_cprobe));
  if (e != cudaSuccess) return cuda_fail(e);
  dims[0] = CPROBE_CTAS;
  dims[1] = CPROBE_TILES;
  dims[2] = CONV_PROBE_PHASES;
  return Y5OBB_OK;
}
#endif
