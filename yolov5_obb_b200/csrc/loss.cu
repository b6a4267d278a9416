// ComputeLoss for the OBB head on the device: build_targets + CIoU box + obj/cls BCE + 180-bin CSL theta BCE,
// forward and backward.  Replaces utils/loss.py:122-192 (__call__), :194-275 (build_targets)
// and utils/metrics.py:201-236 (bbox_iou, CIoU), which run as ~60 small ATen kernels with
// three host syncs per level (boolean-mask indexing) and materialise a dense zero gradient through autograd.
//
//   k_match     one thread per (level, offset k, anchor a, target t) candidate: anchor-ratio test (:237-240)
//               and the 4 neighbour rules (:243-250); candidates are enumerated in the reference's row order
//               (level, k, a, t) so that "last writer wins" on duplicate cells (:159) is the CPU rule
//   cub scan    row ranks and per-level row counts (no host sync)
//   k_rows      one warp per matched row: gather ps = p[b,a,gj,gi,:] (:145), CIoU (:148-152), class BCE
//               (:162-168), theta BCE against the target's CSL row (:171-172); atomicMax picks the winner per cell
//   k_obj       every cell of every level: obj BCE against tobj = clamp(iou(winner), 0) (:155-159,178-179),
//               per-block partial sums
//   k_final     fixed-order reductions, per-level means, gains (:185-189): loss[1], items[4]
//   k_bwd_obj / k_bwd_rows   dL/dp written once: zeros + obj channel for every cell, then the matched rows
// The validation loss (val.py:198-199, y5obb_loss_forward_head) reads no materialised head output: k_head_obj computes the obj
// logits of every cell and k_head_rows the logits of the matched rows from the Detect inputs, into the workspace, and k_rows /
// k_obj read them there (LossK.rows / .obj); everything else is the code above.
// HBM-bound: forward reads one float per cell (32-byte sectors) + 800 bytes per matched row; backward must
// write the dense gradient the autograd contract asks for (B * 64512 * 200 * 4 bytes at 1024x1024).
// Everything is fp32; sums are reduced in a fixed order (deterministic), except gradient accumulation on
// duplicate cells (atomicAdd, order-dependent in the last bit).
#include <cub/device/device_scan.cuh>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstring>

#include <cmath>

#include "common.cuh"

namespace y5obb {
namespace {

constexpr int NOFF = 5;
constexpr int OBJ_THREADS = 256;
constexpr int NL = Y5OBB_LOSS_MAX_LEVELS;

struct LossK {
  const float* p[NL];
  float* grad[NL];
  int H[NL], W[NL];
  long long cell_off[NL + 1];  // prefix of B*na*H*W per level
  float stride[NL];
  float anchors[NL * 3 * 2];
  float balance[NL];
  int nl, B, na, no, nc;
  const float* targets;
  int nt, tcols;
  float anchor_t, cp, cn;
  float hyp_box, hyp_obj, hyp_cls, hyp_theta;
  float cls_pw, obj_pw, theta_pw;
  // workspace
  int* flag;
  int* rank;          // exclusive scan of flag
  int* winner;        // per cell: highest matched row rank (level-local), -1 = none
  float* row_iou;     // per row (global rank)
  float* row_box;     // 1 - ciou
  float* row_cls;     // sum over classes of BCE
  float* row_theta;   // sum over 180 bins of BCE
  double* obj_partial;  // [nl][obj_blocks]
  int obj_blocks[NL];
  long long obj_block_off[NL + 1];
  int ncand;          // nl * 5 * na * nt
  // Circular-Smooth-Label rows (utils/rboxs_utils.py:9-26): csl_mode 0 = 180 floats per target at column 7 (the reference's
  // [nt,187] layout), 1 = column 7 holds the row's rotation index int(90 - angle) (the caller evaluated the truncation in
  // fp64 like the reference), 2 = the index is derived here from theta (column 6, fp32).  Modes 1/2 read gauss[].
  int csl_mode;
  float gauss[180];   // (float)exp(-(j - 90)^2 / (2 sigma^2)), j = 0..179: the un-rotated row of gaussian_label_cpu
  // Where k_rows and k_obj read the logits.  A matched row's no logits start at
  // rows[lvl] + cell_local * row_cell_stride + rank * row_rank_stride; cell i's obj logit is obj[lvl][i * obj_stride + obj_col].
  // The materialised head gives (p, no, 0) and (p, no, 4); the Detect-input path gives its workspace buffers (0, no) and (1, 0).
  const float* rows[NL];
  long long row_cell_stride, row_rank_stride;
  const float* obj[NL];
  long long obj_stride;
  int obj_col;
  void* scan_tmp;
  size_t scan_bytes;
  // Detect-input path (y5obb_loss_forward_head): obj logits [cells] and matched-row logits [ncand, no]
  float* head_obj;
  float* head_rows;
};

// element c of target t's CSL row: gaussian_label_cpu's np.concatenate([y_sig[index:], y_sig[:index]]) = y_sig[(c + index) mod 180]
__device__ __forceinline__ int csl_index(const LossK& L, int t) {
  if (L.csl_mode == 1) return (int)L.targets[(long long)t * L.tcols + 7];
  // rboxs_utils.py:70 angle = theta * 180 / pi + 90 with pi = 3.141592 (fp64), :21 index = int(num_class / 2 - angle)
  const double angle = (double)L.targets[(long long)t * L.tcols + 6] * 180.0 / 3.141592 + 90.0;
  return (int)(90.0 - angle);
}
__device__ __forceinline__ float csl_value(const LossK& L, const float* row, int index, int c) {
  if (L.csl_mode == 0) return row[c];
  int j = (c + index) % 180;
  if (j < 0) j += 180;
  return L.gauss[j];
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// BCEWithLogits with pos_weight (torch: (1 - t) * x + (1 + (pw - 1) * t) * (log1p(exp(-|x|)) + max(-x, 0)))
__device__ __forceinline__ float bce_logits(float x, float t, float pw) {
  const float lw = 1.0f + (pw - 1.0f) * t;
  return (1.0f - t) * x + lw * (log1pf(expf(-fabsf(x))) + fmaxf(-x, 0.0f));
}
__device__ __forceinline__ float bce_logits_grad(float x, float t, float pw) {
  const float s = sigmoidf_(x);
  return s * (1.0f + (pw - 1.0f) * t) - pw * t;
}

struct Cand {
  int lvl, k, a, t;
};
__device__ __forceinline__ Cand decode_cand(const LossK& L, int q) {
  Cand c;
  c.t = q % L.nt;
  int r = q / L.nt;
  c.a = r % L.na;
  r /= L.na;
  c.k = r % NOFF;
  c.lvl = r / NOFF;
  return c;
}

struct TargetGeom {
  float gx, gy, gl, gs;
  int b, cls;
};
__device__ __forceinline__ TargetGeom target_geom(const LossK& L, int lvl, int t) {
  const float* T = L.targets + (long long)t * L.tcols;
  TargetGeom g;
  g.b = (int)T[0];
  g.cls = (int)T[1];
  const float s = L.stride[lvl];
  g.gx = __fdiv_rn(T[2], s);
  g.gy = __fdiv_rn(T[3], s);
  g.gl = __fdiv_rn(T[4], s);
  g.gs = __fdiv_rn(T[5], s);
  return g;
}
__device__ __forceinline__ float frac1(float x) { return x - floorf(x); }  // torch `% 1`

__global__ void k_match(LossK L) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= L.ncand) return;
  const Cand c = decode_cand(L, q);
  const TargetGeom g = target_geom(L, c.lvl, c.t);
  const float aw = L.anchors[(c.lvl * L.na + c.a) * 2], ah = L.anchors[(c.lvl * L.na + c.a) * 2 + 1];
  const float rl = __fdiv_rn(g.gl, aw), rs = __fdiv_rn(g.gs, ah);
  const float m = fmaxf(fmaxf(rl, __fdiv_rn(1.0f, rl)), fmaxf(rs, __fdiv_rn(1.0f, rs)));
  bool ok = m < L.anchor_t;
  if (ok && c.k) {
    const float W = (float)L.W[c.lvl], H = (float)L.H[c.lvl];
    const float gxi = W - g.gx, gyi = H - g.gy;
    switch (c.k) {
      case 1: ok = frac1(g.gx) < 0.5f && g.gx > 1.0f; break;
      case 2: ok = frac1(g.gy) < 0.5f && g.gy > 1.0f; break;
      case 3: ok = frac1(gxi) < 0.5f && gxi > 1.0f; break;
      default: ok = frac1(gyi) < 0.5f && gyi > 1.0f; break;
    }
  }
  L.flag[q] = ok ? 1 : 0;
}

// forward-mode dual numbers over the 4 box logits
struct D4 {
  float v, d[4];
};
__device__ __forceinline__ D4 dconst(float v) { return D4{v, {0.f, 0.f, 0.f, 0.f}}; }
__device__ __forceinline__ D4 operator+(const D4& a, const D4& b) {
  return D4{a.v + b.v, {a.d[0] + b.d[0], a.d[1] + b.d[1], a.d[2] + b.d[2], a.d[3] + b.d[3]}};
}
__device__ __forceinline__ D4 operator-(const D4& a, const D4& b) {
  return D4{a.v - b.v, {a.d[0] - b.d[0], a.d[1] - b.d[1], a.d[2] - b.d[2], a.d[3] - b.d[3]}};
}
__device__ __forceinline__ D4 operator*(const D4& a, const D4& b) {
  D4 r;
  r.v = a.v * b.v;
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
  return r;
}
__device__ __forceinline__ D4 operator/(const D4& a, const D4& b) {
  D4 r;
  const float inv = 1.0f / b.v;
  r.v = a.v * inv;
#pragma unroll
  for (int i = 0; i < 4; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv;
  return r;
}
__device__ __forceinline__ D4 dscale(const D4& a, float s) {
  return D4{a.v * s, {a.d[0] * s, a.d[1] * s, a.d[2] * s, a.d[3] * s}};
}
// torch's rules at ties: minimum / maximum give each side half the derivative, clamp(0) passes it at exactly 0.  Zero box
// logits put the predicted box at (cell + 0.5, anchor), so a target of the anchor's width centred on a cell ties on both edges.
__device__ __forceinline__ D4 dtie(const D4& a, const D4& b) {
  return D4{a.v, {0.5f * (a.d[0] + b.d[0]), 0.5f * (a.d[1] + b.d[1]), 0.5f * (a.d[2] + b.d[2]), 0.5f * (a.d[3] + b.d[3])}};
}
__device__ __forceinline__ D4 dmin(const D4& a, const D4& b) { return a.v < b.v ? a : (b.v < a.v ? b : dtie(a, b)); }
__device__ __forceinline__ D4 dmax(const D4& a, const D4& b) { return a.v > b.v ? a : (b.v > a.v ? b : dtie(a, b)); }
__device__ __forceinline__ D4 dclamp0(const D4& a) { return a.v >= 0.f ? a : dconst(0.f); }
__device__ __forceinline__ D4 datan(const D4& a) {
  const float g = 1.0f / (1.0f + a.v * a.v);
  return D4{atanf(a.v), {a.d[0] * g, a.d[1] * g, a.d[2] * g, a.d[3] * g}};
}

// CIoU of the predicted box (from 4 logits, anchor aw/ah) against the target box (tx, ty, tw, th);
// metrics.py:201-236 with x1y1x2y2=False, CIoU=True, eps=1e-7; alpha carries no gradient (:234-235)
__device__ D4 ciou_dual(const float (&s)[4], float aw, float ah, float tx, float ty, float tw, float th) {
  const float eps = 1e-7f;
  D4 px, py, pw, ph;
  {
    const float s0 = sigmoidf_(s[0]), s1 = sigmoidf_(s[1]), s2 = sigmoidf_(s[2]), s3 = sigmoidf_(s[3]);
    px = D4{s0 * 2.0f - 0.5f, {2.0f * s0 * (1.0f - s0), 0.f, 0.f, 0.f}};
    py = D4{s1 * 2.0f - 0.5f, {0.f, 2.0f * s1 * (1.0f - s1), 0.f, 0.f}};
    const float w2 = s2 * 2.0f, h2 = s3 * 2.0f;
    pw = D4{w2 * w2 * aw, {0.f, 0.f, 8.0f * s2 * s2 * (1.0f - s2) * aw, 0.f}};
    ph = D4{h2 * h2 * ah, {0.f, 0.f, 0.f, 8.0f * s3 * s3 * (1.0f - s3) * ah}};
  }
  const D4 b1x1 = px - dscale(pw, 0.5f), b1x2 = px + dscale(pw, 0.5f);
  const D4 b1y1 = py - dscale(ph, 0.5f), b1y2 = py + dscale(ph, 0.5f);
  const D4 b2x1 = dconst(tx - tw / 2), b2x2 = dconst(tx + tw / 2);
  const D4 b2y1 = dconst(ty - th / 2), b2y2 = dconst(ty + th / 2);
  const D4 inter = dclamp0(dmin(b1x2, b2x2) - dmax(b1x1, b2x1)) * dclamp0(dmin(b1y2, b2y2) - dmax(b1y1, b2y1));
  const D4 w1 = b1x2 - b1x1, h1 = b1y2 - b1y1 + dconst(eps);
  const D4 w2 = b2x2 - b2x1, h2 = b2y2 - b2y1 + dconst(eps);
  const D4 uni = w1 * h1 + w2 * h2 - inter + dconst(eps);
  const D4 iou = inter / uni;
  const D4 cw = dmax(b1x2, b2x2) - dmin(b1x1, b2x1);
  const D4 ch = dmax(b1y2, b2y2) - dmin(b1y1, b2y1);
  const D4 c2 = cw * cw + ch * ch + dconst(eps);
  const D4 dx = b2x1 + b2x2 - b1x1 - b1x2, dy = b2y1 + b2y2 - b1y1 - b1y2;
  const D4 rho2 = dscale(dx * dx + dy * dy, 0.25f);
  const D4 da = datan(w2 / h2) - datan(w1 / h1);
  const D4 v = dscale(da * da, 4.0f / (3.14159265358979323846f * 3.14159265358979323846f));
  const float alpha = v.v / (v.v - iou.v + (1.0f + eps));
  return iou - (rho2 / c2 + dscale(v, alpha));
}

struct RowGeom {
  int lvl, cell_local, b, a, gi, gj, cls, t;
  float tx, ty, tw, th, aw, ah;
};
__device__ __forceinline__ RowGeom row_geom(const LossK& L, int q) {
  const Cand c = decode_cand(L, q);
  const TargetGeom g = target_geom(L, c.lvl, c.t);
  const float ox = c.k == 1 ? 0.5f : (c.k == 3 ? -0.5f : 0.f);
  const float oy = c.k == 2 ? 0.5f : (c.k == 4 ? -0.5f : 0.f);
  const int gi0 = (int)(g.gx - ox), gj0 = (int)(g.gy - oy);  // .long(): truncation toward zero (:263)
  RowGeom r;
  r.lvl = c.lvl;
  r.t = c.t;
  r.b = g.b;
  r.a = c.a;
  r.cls = g.cls;
  r.gi = min(max(gi0, 0), L.W[c.lvl] - 1);  // clamp_ (:267)
  r.gj = min(max(gj0, 0), L.H[c.lvl] - 1);
  r.tx = g.gx - (float)gi0;                 // tbox uses the UNclamped cell (:268)
  r.ty = g.gy - (float)gj0;
  r.tw = g.gl;
  r.th = g.gs;
  r.aw = L.anchors[(c.lvl * L.na + c.a) * 2];
  r.ah = L.anchors[(c.lvl * L.na + c.a) * 2 + 1];
  r.cell_local = ((r.b * L.na + r.a) * L.H[c.lvl] + r.gj) * L.W[c.lvl] + r.gi;
  return r;
}

// level-local rank = global rank - first global rank of the level
__device__ __forceinline__ int level_first_rank(const LossK& L, int lvl) { return L.rank[lvl * NOFF * L.na * L.nt]; }
__device__ __forceinline__ int total_rows(const LossK& L) { return L.rank[L.ncand - 1] + L.flag[L.ncand - 1]; }
__device__ __forceinline__ int level_rows(const LossK& L, int lvl) {
  const int first = level_first_rank(L, lvl);
  const int next = (lvl + 1 < L.nl) ? level_first_rank(L, lvl + 1) : total_rows(L);
  return next - first;
}

__global__ void k_rows(LossK L) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= L.ncand || !L.flag[q]) return;
  const int rank = L.rank[q];
  const RowGeom r = row_geom(L, q);
  if (r.b < 0 || r.b >= L.B) return;  // malformed target row
  const float* ps = L.rows[r.lvl] + (long long)r.cell_local * L.row_cell_stride + (long long)rank * L.row_rank_stride;
  const float* csl = L.targets + (long long)r.t * L.tcols + 7;
  const int csl_i = L.csl_mode ? csl_index(L, r.t) : 0;
  float s_cls = 0.f, s_th = 0.f;
  const int ci = 5 + L.nc;
  if (L.nc > 1)
    for (int c = lane; c < L.nc; c += 32) s_cls += bce_logits(ps[5 + c], c == r.cls ? L.cp : L.cn, L.cls_pw);
  for (int c = lane; c < 180; c += 32) s_th += bce_logits(ps[ci + c], csl_value(L, csl, csl_i, c), L.theta_pw);
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    s_cls += __shfl_xor_sync(0xffffffffu, s_cls, o);
    s_th += __shfl_xor_sync(0xffffffffu, s_th, o);
  }
  if (lane == 0) {
    const float s[4] = {ps[0], ps[1], ps[2], ps[3]};
    const D4 ciou = ciou_dual(s, r.aw, r.ah, r.tx, r.ty, r.tw, r.th);
    L.row_iou[rank] = ciou.v;
    L.row_box[rank] = 1.0f - ciou.v;
    L.row_cls[rank] = s_cls;
    L.row_theta[rank] = s_th;
    atomicMax(&L.winner[L.cell_off[r.lvl] + r.cell_local], rank);  // ranks grow in the reference's row order
  }
}

__global__ void __launch_bounds__(OBJ_THREADS) k_obj(LossK L, int lvl) {
  const long long cells = L.cell_off[lvl + 1] - L.cell_off[lvl];
  const long long i = (long long)blockIdx.x * OBJ_THREADS + threadIdx.x;
  float v = 0.f;
  if (i < cells) {
    const float x = L.obj[lvl][i * L.obj_stride + L.obj_col];
    const int w = L.winner[L.cell_off[lvl] + i];
    const float t = w >= 0 ? fmaxf(L.row_iou[w], 0.f) : 0.f;  // gr = 1.0 (:157-159)
    v = bce_logits(x, t, L.obj_pw);
  }
  __shared__ float red[OBJ_THREADS];
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = OBJ_THREADS / 2; s; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) L.obj_partial[L.obj_block_off[lvl] + blockIdx.x] = (double)red[0];
}

// ---- Detect-input logit source (y5obb_loss_forward_head): the logits the loss reads, computed from the Detect inputs instead of
// being read from a materialised [B, na, H, W, no] head output
struct HeadLevel {
  const __nv_bfloat16* feat;  // NHWC, element strides below
  long long pix, row, img;
  int C;
  const __nv_bfloat16* w;     // [na * no, C]
  const float* bias;          // [na * no]
};
struct HeadK {
  HeadLevel lv[NL];
};
// k_head_rows takes both blocks as its launch parameters (4 KB at most on sm_90)
static_assert(sizeof(LossK) + sizeof(HeadK) <= 4096, "loss kernel parameters exceed the 4 KB launch-parameter limit");

// 8 bf16 (F16: fp16) products of two 16-byte vectors, accumulated in order into acc
template <bool F16>
__device__ __forceinline__ float2 to_float2(const uint32_t& v) {
  if constexpr (F16) return __half22float2(*reinterpret_cast<const __half2*>(&v));
  else return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v));
}
template <bool F16>
__device__ __forceinline__ float dot8(const uint4& x, const uint4& y, float acc) {
  const uint32_t* a = reinterpret_cast<const uint32_t*>(&x);
  const uint32_t* b = reinterpret_cast<const uint32_t*>(&y);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 u = to_float2<F16>(a[i]), v = to_float2<F16>(b[i]);
    acc = fmaf(u.x, v.x, acc);
    acc = fmaf(u.y, v.y, acc);
  }
  return acc;
}

// The logit the loss reads: bias + acc, and for an fp16 plan (F16: fp16 features and weights) that value rounded to fp16, the
// half Detect conv's output that val.py:198-199 widens with `x.float()`
template <bool F16>
__device__ __forceinline__ float head_logit(float bias, float acc) {
  if constexpr (F16) return __half2float(__float2half_rn(bias + acc));
  else return bias + acc;
}

// obj logits of one level: head_obj[cell_off + ((b * na + a) * H + y) * W + x] = bias[a*no+4] + sum_c feat[b,y,x,c] w[a*no+4, c].
// An N = na GEMM bound by the feature read: G lanes (a power of two dividing C/8) share a pixel, every feature byte is read once
// with 16-byte loads, the na weight rows sit in shared memory.
template <bool F16>
__global__ void __launch_bounds__(256) k_head_obj(LossK L, HeadLevel h, int lvl, int G) {
  extern __shared__ uint4 s_w[];  // [na][C / 8]
  const int C8 = h.C / 8;
  for (int i = threadIdx.x; i < L.na * C8; i += blockDim.x) {
    const int a = i / C8;
    s_w[i] = *reinterpret_cast<const uint4*>(h.w + (long long)(a * L.no + 4) * h.C + (i - a * C8) * 8);
  }
  __syncthreads();
  const int H = L.H[lvl], W = L.W[lvl];
  const long long pixels = (long long)L.B * H * W;
  const int lane = threadIdx.x & 31, g = lane & (G - 1);
  float* out = L.head_obj + L.cell_off[lvl];
  // warp-uniform trip count: every lane reaches the shuffles
  const long long step = (long long)gridDim.x * blockDim.x / G;
  for (long long base = ((long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31)) / G; base < pixels; base += step) {
    const long long pix = base + lane / G;
    const bool valid = pix < pixels;
    float acc[3] = {0.f, 0.f, 0.f};
    int b = 0, y = 0, x = 0;
    if (valid) {
      b = (int)(pix / ((long long)H * W));
      const int rem = (int)(pix - (long long)b * H * W);
      y = rem / W;
      x = rem - y * W;
      const __nv_bfloat16* f = h.feat + b * h.img + y * h.row + x * h.pix;
      for (int c8 = g; c8 < C8; c8 += G) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(f + c8 * 8));
#pragma unroll
        for (int a = 0; a < 3; ++a)
          if (a < L.na) acc[a] = dot8<F16>(v, s_w[a * C8 + c8], acc[a]);
      }
    }
    for (int o = G >> 1; o; o >>= 1) {
#pragma unroll
      for (int a = 0; a < 3; ++a) acc[a] += __shfl_xor_sync(0xffffffffu, acc[a], o);
    }
    if (valid && g == 0) {
#pragma unroll
      for (int a = 0; a < 3; ++a)
        if (a < L.na) out[(((long long)b * L.na + a) * H + y) * W + x] = head_logit<F16>(h.bias[a * L.no + 4], acc[a]);
    }
  }
}

// the no logits of every matched row (after k_match and the scan): a gathered GEMV per row, one warp per candidate, written to
// head_rows[rank * no + j] = bias[a*no+j] + sum_c feat[b,gj,gi,c] w[a*no+j, c]
template <bool F16>
__global__ void k_head_rows(LossK L, HeadK hk) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= L.ncand || !L.flag[q]) return;
  const RowGeom r = row_geom(L, q);
  if (r.b < 0 || r.b >= L.B) return;  // k_rows skips the row too
  const HeadLevel& h = hk.lv[r.lvl];
  const int C8 = h.C / 8;
  const __nv_bfloat16* f = h.feat + r.b * h.img + r.gj * h.row + r.gi * h.pix;
  const __nv_bfloat16* w = h.w + (long long)r.a * L.no * h.C;
  const float* bias = h.bias + r.a * L.no;
  float* out = L.head_rows + (long long)L.rank[q] * L.no;
  for (int j0 = 0; j0 < L.no; j0 += 4) {  // the last group of a row whose no % 4 != 0 has fewer than 4 logits
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c8 = lane; c8 < C8; c8 += 32) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(f + c8 * 8));
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (j0 + k < L.no)
          acc[k] = dot8<F16>(v, __ldg(reinterpret_cast<const uint4*>(w + (long long)(j0 + k) * h.C + c8 * 8)), acc[k]);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
    }
    if (lane < 4 && j0 + lane < L.no)
      out[j0 + lane] = head_logit<F16>(bias[j0 + lane], lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3]);
  }
}

// one block; every sum runs in a fixed order
__global__ void __launch_bounds__(256) k_final(LossK L, float* loss, float* items) {
  __shared__ double red[256];
  auto block_sum = [&](auto&& f, long long n) -> double {
    double acc = 0.0;
    for (long long i = threadIdx.x; i < n; i += 256) acc += f(i);
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
  };
  double lbox = 0, lobj = 0, lcls = 0, lth = 0;
  for (int lvl = 0; lvl < L.nl; ++lvl) {
    const int first = level_first_rank(L, lvl);
    const int n = level_rows(L, lvl);
    if (n > 0) {
      lbox += block_sum([&](long long i) { return (double)L.row_box[first + i]; }, n) / n;
      if (L.nc > 1) lcls += block_sum([&](long long i) { return (double)L.row_cls[first + i]; }, n) / ((double)n * L.nc);
      lth += block_sum([&](long long i) { return (double)L.row_theta[first + i]; }, n) / ((double)n * 180.0);
    }
    const long long cells = L.cell_off[lvl + 1] - L.cell_off[lvl];
    const double so = block_sum([&](long long i) { return L.obj_partial[L.obj_block_off[lvl] + i]; }, L.obj_blocks[lvl]);
    lobj += so / (double)cells * L.balance[lvl];
  }
  if (threadIdx.x == 0) {
    const float b = (float)lbox * L.hyp_box, o = (float)lobj * L.hyp_obj, c = (float)lcls * L.hyp_cls,
                t = (float)lth * L.hyp_theta;
    items[0] = b;
    items[1] = o;
    items[2] = c;
    items[3] = t;
    loss[0] = (b + o + c + t) * (float)L.B;
  }
}

// dense gradient: every element of the level is written exactly once here (zeros + obj channel).  The level's cells * no
// floats are walked flat, as float4s (the buffer is 16-byte aligned) and then a scalar tail of (cells * no) % 4; when
// no % 4 != 0 a vector may span the end of one cell's row and the start of the next.
__global__ void k_bwd_obj(LossK L, int lvl, const float* __restrict__ gloss) {
  const long long cells = L.cell_off[lvl + 1] - L.cell_off[lvl];
  const long long n = cells * L.no, nvec = n / 4;
  const float g = gloss[0] * (float)L.B * L.hyp_obj * L.balance[lvl] / (float)cells;
  auto obj_grad = [&](long long cell) {
    const float x = L.p[lvl][cell * L.no + 4];
    const int w = L.winner[L.cell_off[lvl] + cell];
    const float t = w >= 0 ? fmaxf(L.row_iou[w], 0.f) : 0.f;
    return g * bce_logits_grad(x, t, L.obj_pw);
  };
  float* out = L.grad[lvl];
  const long long total = nvec + (n & 3);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (i < nvec) {
      const long long e = 4 * i, cell = e / L.no;
      const int ch = (int)(e - cell * L.no);  // channel of the vector's first element
      // obj (channel 4 of `cell`) is element 4 - ch when ch is 1..4; the next cell's channel 4 lies no >= 185 floats further
      const float v = (ch >= 1 && ch <= 4) ? obj_grad(cell) : 0.f;
      reinterpret_cast<float4*>(out)[i] = make_float4(ch == 4 ? v : 0.f, ch == 3 ? v : 0.f, ch == 2 ? v : 0.f, ch == 1 ? v : 0.f);
    } else {
      const long long e = 4 * nvec + (i - nvec), cell = e / L.no;
      out[e] = e - cell * L.no == 4 ? obj_grad(cell) : 0.f;
    }
  }
}

__global__ void k_bwd_rows(LossK L, const float* __restrict__ gloss) {
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (q >= L.ncand || !L.flag[q]) return;
  const RowGeom r = row_geom(L, q);
  if (r.b < 0 || r.b >= L.B) return;
  const int n = level_rows(L, r.lvl);
  const float up = gloss[0] * (float)L.B;
  const float* ps = L.p[r.lvl] + (long long)r.cell_local * L.no;
  float* gp = L.grad[r.lvl] + (long long)r.cell_local * L.no;
  const float* csl = L.targets + (long long)r.t * L.tcols + 7;
  const int csl_i = L.csl_mode ? csl_index(L, r.t) : 0;
  const int ci = 5 + L.nc;
  if (L.nc > 1) {
    const float gc = up * L.hyp_cls / ((float)n * (float)L.nc);
    for (int c = lane; c < L.nc; c += 32)
      atomicAdd(gp + 5 + c, gc * bce_logits_grad(ps[5 + c], c == r.cls ? L.cp : L.cn, L.cls_pw));
  }
  const float gt = up * L.hyp_theta / ((float)n * 180.0f);
  for (int c = lane; c < 180; c += 32)
    atomicAdd(gp + ci + c, gt * bce_logits_grad(ps[ci + c], csl_value(L, csl, csl_i, c), L.theta_pw));
  if (lane == 0) {
    const float s[4] = {ps[0], ps[1], ps[2], ps[3]};
    const D4 ciou = ciou_dual(s, r.aw, r.ah, r.tx, r.ty, r.tw, r.th);
    const float gb = -up * L.hyp_box / (float)n;  // d(1 - ciou)
#pragma unroll
    for (int i = 0; i < 4; ++i) atomicAdd(gp + i, gb * ciou.d[i]);
  }
}

int fill(LossK& L, const y5obb_loss_desc* d, void* ws, size_t ws_bytes, size_t* need, bool head = false) {
  if (!d || d->nl < 1 || d->nl > NL || d->B < 1 || d->na < 1 || d->na > 3 || d->nt < 0) return Y5OBB_EINVAL;
  if (d->no != d->nc + 5 + 180) return Y5OBB_EINVAL;
  if (d->tcols != 7 && d->tcols != 8 && d->tcols < 7 + 180) return Y5OBB_EINVAL;
  memset(&L, 0, sizeof(L));
  L.csl_mode = d->tcols == 7 ? 2 : (d->tcols == 8 ? 1 : 0);
  {
    const double sig = d->csl_sigma > 0 ? (double)d->csl_sigma : 2.0;  // hyp['csl_radius'] (hyp.finetune_dota.yaml:34)
    for (int j = 0; j < 180; ++j) {
      const double x = (double)j - 90.0;
      L.gauss[j] = (float)std::exp(-(x * x) / (2.0 * sig * sig));
    }
  }
  L.nl = d->nl;
  L.B = d->B;
  L.na = d->na;
  L.no = d->no;
  L.nc = d->nc;
  L.targets = d->targets;
  L.nt = d->nt;
  L.tcols = d->tcols;
  L.anchor_t = d->anchor_t;
  L.cp = d->cp;
  L.cn = d->cn;
  L.hyp_box = d->hyp_box;
  L.hyp_obj = d->hyp_obj;
  L.hyp_cls = d->hyp_cls;
  L.hyp_theta = d->hyp_theta;
  L.cls_pw = d->cls_pw;
  L.obj_pw = d->obj_pw;
  L.theta_pw = d->theta_pw;
  long long cells = 0;
  long long blocks = 0;
  for (int i = 0; i < d->nl; ++i) {
    L.p[i] = d->p[i];
    L.grad[i] = d->grad[i];
    L.H[i] = d->H[i];
    L.W[i] = d->W[i];
    L.stride[i] = d->stride[i];
    L.balance[i] = d->balance[i];
    L.cell_off[i] = cells;
    cells += (long long)d->B * d->na * d->H[i] * d->W[i];
    L.obj_blocks[i] = (int)(((long long)d->B * d->na * d->H[i] * d->W[i] + OBJ_THREADS - 1) / OBJ_THREADS);
    L.obj_block_off[i] = blocks;
    blocks += L.obj_blocks[i];
  }
  L.cell_off[d->nl] = cells;
  for (int i = 0; i < d->nl; ++i) L.rows[i] = L.obj[i] = d->p[i];
  L.row_cell_stride = L.obj_stride = d->no;
  L.row_rank_stride = 0;
  L.obj_col = 4;
  L.obj_block_off[d->nl] = blocks;
  for (int i = 0; i < NL * 3 * 2; ++i) L.anchors[i] = d->anchors[i];
  L.ncand = d->nl * NOFF * d->na * d->nt;
  const int nc1 = L.ncand > 0 ? L.ncand : 1;
  Carver c(ws);
  L.flag = c.take<int>(nc1);
  L.rank = c.take<int>(nc1);
  L.winner = c.take<int>(cells);
  L.row_iou = c.take<float>(nc1);
  L.row_box = c.take<float>(nc1);
  L.row_cls = c.take<float>(nc1);
  L.row_theta = c.take<float>(nc1);
  L.obj_partial = c.take<double>(blocks);
  size_t scan_bytes = 0;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, nc1, 0);
  if (e != cudaSuccess || scan_bytes == 0) {
    (void)cudaGetLastError();
    scan_bytes = (1u << 20);
  }
  L.scan_tmp = c.take<char>(scan_bytes);
  L.scan_bytes = scan_bytes;
  if (head) {
    L.head_obj = c.take<float>(cells);
    L.head_rows = c.take<float>((size_t)nc1 * d->no);
    for (int i = 0; i < d->nl; ++i) {
      L.rows[i] = L.head_rows;
      L.obj[i] = L.head_obj + L.cell_off[i];
    }
    L.row_cell_stride = 0;
    L.row_rank_stride = d->no;
    L.obj_stride = 1;
    L.obj_col = 0;
  }
  *need = c.used() + 256;
  if (ws && *need > ws_bytes) return Y5OBB_EWORKSPACE;
  return Y5OBB_OK;
}

// The forward shared by both logit sources; hk != nullptr computes the logits from the Detect inputs first (f16: fp16
// features and weights, logits rounded to fp16).
int forward(LossK& L, const HeadK* hk, float* loss1, float* items4, cudaStream_t st, bool f16 = false) {
  if (L.nt > 0 && !L.targets) return Y5OBB_EINVAL;
  Y5_CUDA(cudaMemsetAsync(L.winner, 0xFF, (size_t)L.cell_off[L.nl] * sizeof(int), st));
  if (L.ncand > 0) {
    k_match<<<(L.ncand + 255) / 256, 256, 0, st>>>(L);
    Y5_LAUNCH_CHECK();
    Y5_CUDA(cub::DeviceScan::ExclusiveSum(L.scan_tmp, L.scan_bytes, L.flag, L.rank, L.ncand, st));
    const long long threads = (long long)L.ncand * 32;
    if (hk) {
      (f16 ? k_head_rows<true> : k_head_rows<false>)<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(L, *hk);
      Y5_LAUNCH_CHECK();
    }
    k_rows<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(L);
    Y5_LAUNCH_CHECK();
  } else {
    // no targets: rank/flag single dummy entry = 0 so that level_rows() == 0
    Y5_CUDA(cudaMemsetAsync(L.flag, 0, sizeof(int), st));
    Y5_CUDA(cudaMemsetAsync(L.rank, 0, sizeof(int), st));
  }
  for (int lvl = 0; lvl < L.nl; ++lvl) {
    if (hk) {
      const HeadLevel& h = hk->lv[lvl];
      const int C8 = h.C / 8;
      int G = 1;
      while (G < 32 && C8 % (2 * G) == 0) G *= 2;
      const long long threads = (long long)L.B * L.H[lvl] * L.W[lvl] * G;
      const int grid = (int)std::min<long long>((threads + 255) / 256, (long long)sm_count() * 8);
      (f16 ? k_head_obj<true> : k_head_obj<false>)<<<grid, 256, (size_t)L.na * C8 * sizeof(uint4), st>>>(L, h, lvl, G);
      Y5_LAUNCH_CHECK();
    }
    k_obj<<<L.obj_blocks[lvl], OBJ_THREADS, 0, st>>>(L, lvl);
    Y5_LAUNCH_CHECK();
  }
  if (L.ncand == 0) L.ncand = 1;  // k_final reads rank[ncand-1] + flag[ncand-1]
  k_final<<<1, 256, 0, st>>>(L, loss1, items4);
  Y5_LAUNCH_CHECK();
  return Y5OBB_OK;
}

// Checks the Detect inputs and gives the loss description they imply: H / W from the features, no materialised logits.
int head_desc(const y5obb_loss_desc* d, const y5obb_loss_head* h, y5obb_loss_desc* dd, HeadK* hk) {
  if (!d || !h || d->nl < 1 || d->nl > NL || d->na < 1 || d->na > 3 || d->no < 1) return Y5OBB_EINVAL;
  *dd = *d;
  memset(hk, 0, sizeof(*hk));
  for (int i = 0; i < d->nl; ++i) {
    const int C = h->C[i], H = h->H[i], W = h->W[i];
    const long long pix = h->pix_stride[i], row = h->row_stride[i], img = h->img_stride[i];
    if (!h->feat[i] || !h->w[i] || !h->bias[i]) return Y5OBB_EINVAL;
    if (C < 8 || C % 8 || H < 1 || W < 1) return Y5OBB_EINVAL;
    if (pix < C || pix % 8 || row < (long long)W * pix || row % 8 || img < (long long)H * row || img % 8) return Y5OBB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(h->feat[i]) | reinterpret_cast<uintptr_t>(h->w[i])) & 15) return Y5OBB_EINVAL;
    dd->p[i] = nullptr;
    dd->grad[i] = nullptr;
    dd->H[i] = H;
    dd->W[i] = W;
    hk->lv[i] = HeadLevel{reinterpret_cast<const __nv_bfloat16*>(h->feat[i]), pix, row, img, C,
                          reinterpret_cast<const __nv_bfloat16*>(h->w[i]), h->bias[i]};
  }
  return Y5OBB_OK;
}

}  // namespace
}  // namespace y5obb

using namespace y5obb;

extern "C" {

size_t y5obb_loss_workspace_bytes(const y5obb_loss_desc* d) {
  LossK L;
  size_t need = 0;
  if (fill(L, d, nullptr, 0, &need) != Y5OBB_OK) return 0;
  return need;
}

int y5obb_loss_forward(const y5obb_loss_desc* d, float* loss1, float* items4, void* workspace, size_t workspace_bytes,
                       void* stream) {
  if (!loss1 || !items4 || !workspace) return Y5OBB_EINVAL;
  LossK L;
  size_t need = 0;
  int rc = fill(L, d, workspace, workspace_bytes, &need);
  if (rc) return rc;
  for (int i = 0; i < L.nl; ++i)
    if (!L.p[i]) return Y5OBB_EINVAL;
  return forward(L, nullptr, loss1, items4, (cudaStream_t)stream);
}

size_t y5obb_loss_head_workspace_bytes(const y5obb_loss_desc* d, const y5obb_loss_head* head) {
  y5obb_loss_desc dd;
  HeadK hk;
  LossK L;
  size_t need = 0;
  if (head_desc(d, head, &dd, &hk) != Y5OBB_OK || fill(L, &dd, nullptr, 0, &need, true) != Y5OBB_OK) return 0;
  return need;
}

static int loss_forward_head(bool f16, const y5obb_loss_desc* d, const y5obb_loss_head* head, float* loss1, float* items4,
                             void* workspace, size_t workspace_bytes, void* stream) {
  if (!loss1 || !items4 || !workspace) return Y5OBB_EINVAL;
  y5obb_loss_desc dd;
  HeadK hk;
  int rc = head_desc(d, head, &dd, &hk);
  if (rc) return rc;
  LossK L;
  size_t need = 0;
  rc = fill(L, &dd, workspace, workspace_bytes, &need, true);
  if (rc) return rc;
  return forward(L, &hk, loss1, items4, (cudaStream_t)stream, f16);
}

int y5obb_loss_forward_head(const y5obb_loss_desc* d, const y5obb_loss_head* head, float* loss1, float* items4,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return loss_forward_head(false, d, head, loss1, items4, workspace, workspace_bytes, stream);
}

int y5obb_loss_forward_head_f16(const y5obb_loss_desc* d, const y5obb_loss_head* head, float* loss1, float* items4,
                                void* workspace, size_t workspace_bytes, void* stream) {
  return loss_forward_head(true, d, head, loss1, items4, workspace, workspace_bytes, stream);
}

int y5obb_loss_backward(const y5obb_loss_desc* d, const float* grad_loss, void* workspace, size_t workspace_bytes,
                        void* stream) {
  if (!grad_loss || !workspace) return Y5OBB_EINVAL;
  LossK L;
  size_t need = 0;
  int rc = fill(L, d, workspace, workspace_bytes, &need);
  if (rc) return rc;
  for (int i = 0; i < L.nl; ++i)
    if (!L.p[i] || !L.grad[i] || (reinterpret_cast<uintptr_t>(L.grad[i]) & 15)) return Y5OBB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int real_cand = L.ncand;
  if (L.ncand == 0) L.ncand = 1;
  for (int lvl = 0; lvl < L.nl; ++lvl) {
    const long long total = (L.cell_off[lvl + 1] - L.cell_off[lvl]) * L.no / 4 + 3;  // >= k_bwd_obj's float4s + tail
    const int grid = (int)std::min<long long>((total + 255) / 256, (long long)sm_count() * 32);
    k_bwd_obj<<<grid, 256, 0, st>>>(L, lvl, grad_loss);
    Y5_LAUNCH_CHECK();
  }
  if (real_cand > 0) {
    const long long threads = (long long)real_cand * 32;
    k_bwd_rows<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(L, grad_loss);
    Y5_LAUNCH_CHECK();
  }
  return Y5OBB_OK;
}

}  // extern "C"
