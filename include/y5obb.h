/* y5obb.h — C ABI of the H100-native (sm_90a) yolov5_obb hot path (liby5obb.so).
 *
 * Plain pointers and sizes only; every pointer is a DEVICE pointer unless its name ends in _host.
 * All entry points are asynchronous on `stream` (a cudaStream_t passed as void*) unless stated, never
 * call cudaDeviceSynchronize, and return 0 on success or a Y5OBB_E* code (the Python shims raise
 * RuntimeError on != 0, as the reference's AT_ASSERTM / AT_CUDA_CHECK do).
 *
 * Each declaration cites the reference interface it replaces (paths relative to the yolov5_obb source tree).
 */
#ifndef Y5OBB_H_
#define Y5OBB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define Y5OBB_OK 0
#define Y5OBB_EINVAL 1     /* bad argument (null pointer, negative size, unsupported shape) */
#define Y5OBB_EWORKSPACE 2 /* workspace too small: call the matching *_workspace_bytes */
#define Y5OBB_ECUDA 3      /* a CUDA call failed; y5obb_last_cuda_error() has the cudaError_t */
#define Y5OBB_EARCH 4      /* device is not sm_90 */

/* ---- library ------------------------------------------------------------------------------- */
int y5obb_abi_version(void);            /* bumps when a signature changes */
int y5obb_last_cuda_error(void);        /* cudaError_t of the last failing CUDA call on this thread */
const char* y5obb_build_info(void);     /* "liby5obb sm_90a <date> <time>" */

/* ---- rotated NMS ---------------------------------------------------------------------------
 * Replaces  utils/nms_rotated/src/nms_rotated_ext.cpp:25-39  (nms_rotated(dets, scores, thr))
 *           utils/nms_rotated/src/nms_rotated_cuda.cu:71-134 (sort, 64x64 IoU bit-matrix, D2H, host scan)
 *           utils/nms_rotated/nms_rotated_wrapper.py:26-42   (min(w,h) < 0.001 pre-filter)
 * Everything — sort, IoU tiles, greedy scan, compaction — runs on the device; nothing is copied to
 * the host.
 *
 * flags */
#define Y5OBB_NMS_STRICT_GT 1   /* suppress if IoU >  thr (reference CUDA, nms_rotated_cuda.cu:60); else */
                                /* suppress if IoU >= thr (reference CPU, nms_rotated_cpu.cpp:55)         */
#define Y5OBB_NMS_DROP_SMALL 2  /* boxes with min(w,h) < 0.001 never enter NMS (nms_rotated_wrapper.py:32) */
#define Y5OBB_NMS_NO_CLASS_SPLIT 4  /* y5obb_nms_obb_f32 only: run ONE greedy pass per image over the class-offset boxes
                                       exactly as general.py:849-853 does, instead of independent (image, class)
                                       passes.  The split is the default when classes are offset (not agnostic); it
                                       gives the same rows whenever boxes of different classes cannot overlap, which
                                       the kernel verifies per box (r + max(|cx|,|cy|) < max_wh/2 - 8); if the test
                                       fails counts[batch] comes back as -2 and the caller re-runs with this flag */

#define Y5OBB_NMS_COMPACT_PRED 8     /* y5obb_nms_obb_f32 only: `pred` holds the Detect epilogue's compact records
                                       [batch, anchors, ((nc + 6) + 3) / 4 * 4] = (cx, cy, w, h, obj, cls[nc], theta index, pad)
                                       instead of the [batch, anchors, no] tensor (y5obb_conv_desc.det_decode = 2).  The theta
                                       index is the first maximum of the 180 theta LOGITS (= torch.max over their sigmoids,
                                       utils/general.py:822, whenever those are distinct) */

/* Workspace needed for n_total boxes over n_images images with at most max_per_image boxes in any one
 * image (pass n_total if unknown). */
size_t y5obb_nms_workspace_bytes(int64_t n_total, int64_t n_images, int64_t max_per_image);

/* One NMS problem.  dets5 [n,5] = (cx, cy, w, h, theta_rad) fp32 row-major, scores [n] fp32.
 * keep_out [n] int64 receives indices into dets5 in descending-score order (ties: lower index first);
 * n_keep_out [1] int64 receives the count. */
int y5obb_nms_rotated_f32(const float* dets5, const float* scores, int64_t n, float iou_thr, int flags,
                          int64_t* keep_out, int64_t* n_keep_out,
                          void* workspace, size_t workspace_bytes, void* stream);

/* n_images independent problems in one launch sequence.  image_ids [n_total] int32 in [0, n_images)
 * (any order).  Image b's kept indices (into dets5) are written in descending-score order to
 * keep_out[seg_off_out[b] .. seg_off_out[b] + n_keep_out[b]); seg_off_out has n_images + 1 entries.
 * max_keep > 0 stops each image after that many keeps (non_max_suppression_obb's max_det,
 * utils/general.py:854-855); 0 = unlimited. */
int y5obb_nms_rotated_batched_f32(const float* dets5, const float* scores, const int32_t* image_ids,
                                  int64_t n_total, int64_t n_images, int64_t max_per_image,
                                  float iou_thr, int flags, int64_t max_keep,
                                  int64_t* keep_out, int64_t* n_keep_out, int64_t* seg_off_out,
                                  void* workspace, size_t workspace_bytes, void* stream);

/* Profiling aid for the single-pass NMS (y5obb_nms_rotated[_batched]_f32): with timing on, CUDA events are recorded on the
 * caller's stream between the stages; y5obb_nms_debug_stage_ms then returns {key+radix sort, segments/plan/prep, k_tiles
 * (pairwise IoU bit matrix), k_reduce (greedy scan + compaction)} of the most recent call in milliseconds. */
int y5obb_nms_debug_stage_timing(int on);
int y5obb_nms_debug_stage_ms(float* ms4);

/* Pairwise rotated IoU of n independent pairs (a[i], b[i]), each 5 floats.  Device restatement of
 * utils/nms_rotated/src/box_iou_rotated_utils.h:334-360 (single_box_iou_rotated<float>). */
int y5obb_rbox_iou_pairs_f32(const float* a5, const float* b5, float* iou_out, int64_t n, void* stream);

/* non_max_suppression_obb on the device (utils/general.py:772-862): conf filter, conf = obj*cls, theta =
 * (argmax(180) - 90)/180*3.141592, multi-label expansion, optional class filter (class_mask bit j = class j
 * allowed; ~0 = all), per-image top-max_nms clamp, class offset cls*max_wh on the centre, rotated NMS,
 * max_det.  pred is the Detect eval output [batch, anchors, no] fp32.  Output: out7 [batch, max_det, 7] rows
 * (cx, cy, l, s, theta, conf, cls) in descending-score order, counts [batch + 1] int64 = rows per image, then
 * the total number of candidates found (if > max_candidates the result is incomplete: call again with a
 * larger max_candidates; the Python shim does).  Nothing is synchronised or copied to the host. */
size_t y5obb_nms_obb_workspace_bytes(int64_t batch, int64_t anchors, int64_t max_candidates, int64_t max_nms);
int y5obb_nms_obb_f32(const float* pred, int64_t batch, int64_t anchors, int no, int nc, float conf_thres,
                      float iou_thres, uint64_t class_mask, int agnostic, int multi_label, int max_det, int max_nms,
                      float max_wh, int flags, int64_t max_candidates, float* out7, int64_t* counts,
                      void* workspace, size_t workspace_bytes, void* stream);


/* ---- convolution (wgmma implicit GEMM) -----------------------------------------------------
 * Replaces the cuDNN/ATen calls behind models/common.py:37-49 (Conv.forward_fuse = conv + folded-BN
 * bias + SiLU), :94-104 (Bottleneck residual), :267-274 (Concat, as a channel-offset store),
 * nn.Upsample(2x nearest) (models/yolov5*.yaml head) and models/yolo.py:49-81 (Detect).
 * Activations are NHWC bf16; a tensor argument is a channel SLICE of a wider buffer: `ptr` points at
 * the slice's first channel of pixel 0 and `*_pix_stride` is the element distance between pixels.
 * Weights are bf16 packed [KH*KW][cout_pad][cin_pad] (K-major), bias fp32 [cout_pad + 32]
 * (the epilogue reads it in 32-wide chunks); the paddings and
 * the tile shape come from y5obb_conv_tiling so that host packing and kernel agree. */
typedef struct y5obb_conv y5obb_conv_t;

#define Y5OBB_CONV_MODE_CONV 0    /* bf16 NHWC output (+ optional residual / 2x up-sampled copy) */
#define Y5OBB_CONV_MODE_DETECT 1  /* Detect head: fp32 [B, rows, no] output, optional sigmoid+decode */

#define Y5OBB_CONV_NO_ROWSHIFT 1   /* flags: force one TMA load per tap (debug / A-B comparison) */
#define Y5OBB_CONV_NO_RESIDENT 2   /* flags: always stream the weight tiles */
#define Y5OBB_CONV_BIAS_HALVED 8    /* flags: REQUIRED when act = 1: `bias` holds 0.5 * b (SiLU is evaluated as h + h*tanh(h), h = x/2) */
#define Y5OBB_CONV_NO_GROUP 16      /* flags: one (tap, K-chunk) unit per pipeline stage */
#define Y5OBB_CONV_NO_PAIRW 4      /* flags: stride-2 convs use TMA element strides along W instead of the pixel-pair view */
#define Y5OBB_CONV_NO_PDL 32       /* flags: plain stream-ordered launch (default: programmatic dependent launch - the kernel's
                                      prologue overlaps the previous kernel's tail and it waits, griddepcontrol.wait, before its
                                      first global-memory access; also switched off by the environment variable Y5OBB_NO_PDL=1) */
#define Y5OBB_CONV_ONE_CTA 64      /* flags: one CTA per SM even for N tiles <= 96 (default: two when the plan fits half of
                                      the shared memory; debug / A-B comparison) */

typedef struct {
  const void* in;            /* bf16 NHWC slice */
  int64_t in_pix_stride;     /* elements between horizontally adjacent input pixels */
  int64_t in_row_stride;     /* elements between image rows (0 = Win * in_pix_stride) */
  int64_t in_img_stride;     /* elements between images     (0 = Hin * in_row_stride) */
  int B, Hin, Win, Cin;      /* Cin may exceed in_pix_stride: overlapping windows (the stem's merged-kw view) */
  int hbm_cin;               /* channels really read per pixel, for the byte accounting (0 = Cin) */
  const void* w;             /* packed weights */
  const float* bias;
  int Cout, KH, KW, stride, pad_h, pad_w;
  int mode, act;             /* act: 0 = identity, 1 = SiLU */
  int flags;
  void* out;                 /* bf16 NHWC slice (MODE_CONV) */
  int64_t out_pix_stride;
  const void* res;           /* optional residual slice added after the activation (Bottleneck.add) */
  int64_t res_pix_stride;
  void* out2x;               /* optional second destination receiving the 2x nearest up-sampled result */
  int64_t out2x_pix_stride;
  float* det_out;            /* MODE_DETECT: fp32, row = b*det_rows_per_image + det_row_off + (a*H + h)*W + w */
  int64_t det_rows_per_image, det_row_off;
  int det_no;                /* outputs per anchor (nc + 5 + 180) */
  int det_decode;            /* 1: sigmoid + xy/wh decode (eval branch, yolo.py:71-74); 0: raw logits (train) */
  float det_stride;          /* level stride in pixels */
  float det_anchor[6];       /* anchor (w,h) in pixels for the 3 anchors of this level */
  /* optional output geometry (MODE_CONV only; all 0 = derived / dense): the output has out_h x out_w pixels (rows and
     columns of the input read beyond its extent are zero), and out / res pixels (b, h, w) live at
     b * img_stride + h * row_stride + w * pix_stride (elements).  Used by the data gradient of stride-2 convolutions:
     each output-pixel parity class is a 1- or 2-tap stride-1 convolution of dz written to every other pixel. */
  int out_h, out_w;
  int64_t out_row_stride, out_img_stride, res_row_stride, res_img_stride;
  /* optional de-scale of a test-time-augmentation branch (MODE_DETECT with det_decode 1 or 2; 0 = off): after the decode,
     x, y, w and h are multiplied by det_inv_scale (the fp32 reciprocal of the fp32 scale, which is what ATen's `p[..., :4] /= s`
     computes on CUDA), then x = det_flip_w - x when det_flip_w > 0 (the left-right de-flip, det_flip_w = image width);
     _descale_pred, models/yolo.py:183-198.  The angle columns are left as they are, as the reference leaves them. */
  int det_descale;
  float det_inv_scale, det_flip_w;
} y5obb_conv_desc;

int y5obb_conv_tiling(int cin, int cout, int mode, int det_no, int* block_k, int* block_n, int* cin_pad,
                      int* cout_pad, int* n_tiles_n);
/* Builds TMA descriptors and launch geometry for fixed buffers (host call, no stream work). */
int y5obb_conv_create(const y5obb_conv_desc* desc, y5obb_conv_t** out);
int y5obb_conv_run(const y5obb_conv_t* conv, void* stream);
int y5obb_conv_info(const y5obb_conv_t* conv, double* flops, double* hbm_bytes, int* grid, int* block_n,
                    int* block_k, int* stages);
/* The rest of the launch plan: CTAs resident per SM (1 or 2), weights resident in shared memory (0/1), row-shift A stages
   (0/1) and (tap, K-chunk) units per pipeline stage.  Any pointer may be NULL. */
int y5obb_conv_schedule(const y5obb_conv_t* conv, int* ctas_per_sm, int* resident, int* rowshift, int* group);
void y5obb_conv_destroy(y5obb_conv_t* conv);

/* ---- HBM-bound helpers around the conv stack -------------------------------------------------
 * y5obb_stem_s2d: NCHW fp32 image [B,3,H,W] -> 2x2 space-to-depth NHWC bf16 [B,H/2,W/2,16] (channel
 * (dy*2+dx)*3 + c, 4 zero channels; rows hold pad_cols untouched (zero) pixels on each side), so that the stem Conv(3, c, 6, 2, 2) of models/yolov5*.yaml (layer 0,
 * models/common.py:37-49) becomes a 3x3/s1/p1 conv for the tensor-core kernel.
 * y5obb_sppf_pool: SPPF's three chained MaxPool2d(5,1,2) (models/common.py:181-196) in one pass over
 * channels [0,C) of an NHWC bf16 buffer, results at channel offsets C, 2C, 3C (replaces torch.cat). */
int y5obb_stem_s2d(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream);
/* same for a uint8 image, with the caller-side `/ 255` (train.py:299, val.py:187-188) folded in */
int y5obb_stem_s2d_u8(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int pad_cols, void* stream);
/* y5obb_scale_img_s2d: scale_img (utils/torch_utils.py:239-249) of one test-time-augmentation branch straight into the stem
 * input: F.interpolate(x or x.flip(3), size=(h, w), mode='bilinear', align_corners=False) with ATen's CUDA arithmetic
 * (upsample_bilinear2d_out_frame<float, float>, its fused products restated), then F.pad right / bottom with pad_value to
 * Hp x Wp, written in y5obb_stem_s2d's layout [B, Hp/2, Wp/2 + 2*pad_cols, 16].  x [B, 3, H, W]; flip_lr != 0 resamples
 * x.flip(3); h <= Hp, w <= Wp, Hp and Wp even.  The pad_cols columns are not written. */
int y5obb_scale_img_s2d(const float* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                        int flip_lr, float pad_value, int pad_cols, void* stream);
/* same for a uint8 image: each input value is (float)u / 255.0f, as in y5obb_stem_s2d_u8 */
int y5obb_scale_img_s2d_u8(const uint8_t* x_nchw, void* out_nhwc16, int B, int H, int W, int h, int w, int Hp, int Wp,
                           int flip_lr, float pad_value, int pad_cols, void* stream);
int y5obb_sppf_pool(void* buf, int64_t pix_stride, int B, int H, int W, int C, void* stream);

/* ---- loss ------------------------------------------------------------------------------------
 * Replaces utils/loss.py:122-192 (ComputeLoss.__call__), :194-275 (build_targets) and utils/metrics.py:201-236
 * (bbox_iou, CIoU).  p[i]: Detect training outputs [B, na, H_i, W_i, no] fp32 (models/yolo.py:65);
 * targets [nt, tcols] fp32 rows (img, cls, cx, cy, l, s, theta, csl[180]) in pixels (utils/datasets.py:643-659).
 * Compact targets (SURVEY 8f rank 2: ship 7-8 floats per box over PCIe instead of 187): tcols == 8 -> column 7 is the row's
 * rotation index int(90 - angle) of utils/rboxs_utils.py:21, evaluated by the caller in fp64 like the reference, and the kernel
 * rebuilds the Circular-Smooth-Label row from it (identical loss, the truncation being the only ill-conditioned step);
 * tcols == 7 -> the index is derived in the kernel from theta (column 6): equal to the reference unless fp32 rounding of
 * theta moves angle across an integer (exact multiples of 1 degree can land on either side).
 * loss1[0] = (lbox + lobj + lcls + ltheta) * B, items4 = (lbox, lobj, lcls, ltheta) after the hyp gains
 * (loss.py:185-192).  backward writes dLoss/dp[i] * grad_loss[0] into grad[i] (dense, same shape as p[i]); it
 * must be given the workspace its forward filled.  Duplicate (b,a,gj,gi) cells: the highest source row wins
 * tobj, as sequential CPU index assignment does (loss.py:159). */
#define Y5OBB_LOSS_MAX_LEVELS 4    /* P3-P5 (yolov5{n,s,m,l,x}) and P3-P6 (models/hub/yolov5{n,s,m,l,x}6); nl <= this */
typedef struct {
  const float* p[Y5OBB_LOSS_MAX_LEVELS];
  float* grad[Y5OBB_LOSS_MAX_LEVELS];      /* backward only */
  int H[Y5OBB_LOSS_MAX_LEVELS], W[Y5OBB_LOSS_MAX_LEVELS];
  float stride[Y5OBB_LOSS_MAX_LEVELS];
  float anchors[Y5OBB_LOSS_MAX_LEVELS * 3 * 2];  /* Detect.anchors: [nl][na][2] in grid units, na <= 3 */
  float balance[Y5OBB_LOSS_MAX_LEVELS];    /* {4.0, 1.0, 0.4}; four levels {4.0, 1.0, 0.25, 0.06} (loss.py:114) */
  int nl, B, na, no, nc;
  const float* targets;
  int nt, tcols;
  float anchor_t, cp, cn;    /* hyp['anchor_t']; smooth_BCE targets (loss.py:107) */
  float hyp_box, hyp_obj, hyp_cls, hyp_theta;  /* already rescaled as train.py:249-252 does */
  float cls_pw, obj_pw, theta_pw;              /* BCEWithLogitsLoss pos_weight (loss.py:99-101) */
  float csl_sigma;                             /* hyp['csl_radius'] for compact targets (tcols 7 / 8); 0 = 2.0 */
} y5obb_loss_desc;

size_t y5obb_loss_workspace_bytes(const y5obb_loss_desc* desc);
int y5obb_loss_forward(const y5obb_loss_desc* desc, float* loss1, float* items4, void* workspace,
                       size_t workspace_bytes, void* stream);
int y5obb_loss_backward(const y5obb_loss_desc* desc, const float* grad_loss, void* workspace,
                        size_t workspace_bytes, void* stream);

/* The validation loss of val.py:198-199 (compute_loss(train_out)[1] for an eval forward; utils/loss.py:122-192) without the
 * materialised head output: the logits the loss reads are computed from the Detect inputs.  Per level, the na obj logits of
 * every cell (an N = na GEMM reading each feature once) and the no logits of every matched row (a gathered GEMV), accumulated
 * in fp32 as bias + sum_c feat * w; everything after that (matching, CIoU, class / theta BCE, obj BCE, reductions) is
 * y5obb_loss_forward's own code, so loss1 / items4 are bit-identical to y5obb_loss_forward on logits equal to these.
 * desc.p and desc.grad are ignored and desc.H / desc.W are replaced by the feature shapes.  Forward only.
 * Y5OBB_EINVAL when a pointer is null, C % 8 != 0, a stride is smaller than the extent it spans or not a multiple of 8
 * elements, or feat / w is not 16-byte aligned.  The workspace holds the obj logits (4 bytes per cell) and
 * nl * 5 * na * nt rows of no floats besides y5obb_loss_forward's own. */
typedef struct {
  const void* feat[Y5OBB_LOSS_MAX_LEVELS];   /* bf16 NHWC Detect input of level i (Detect.f[i]'s output) */
  int64_t pix_stride[Y5OBB_LOSS_MAX_LEVELS], row_stride[Y5OBB_LOSS_MAX_LEVELS],
      img_stride[Y5OBB_LOSS_MAX_LEVELS];     /* element strides of pixels, rows and images */
  int H[Y5OBB_LOSS_MAX_LEVELS], W[Y5OBB_LOSS_MAX_LEVELS], C[Y5OBB_LOSS_MAX_LEVELS];  /* feature shape; C % 8 == 0 */
  const void* w[Y5OBB_LOSS_MAX_LEVELS];      /* bf16 [na * no, C]: Detect.m[i].weight */
  const float* bias[Y5OBB_LOSS_MAX_LEVELS];  /* fp32 [na * no]:    Detect.m[i].bias */
} y5obb_loss_head;

size_t y5obb_loss_head_workspace_bytes(const y5obb_loss_desc* desc, const y5obb_loss_head* head);
int y5obb_loss_forward_head(const y5obb_loss_desc* desc, const y5obb_loss_head* head, float* loss1, float* items4,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- post-NMS geometry and CSL targets (one thread per box, fp32, separately rounded ops) -------
 * rbox2poly: utils/rboxs_utils.py:106-126 — [n,5] (cx,cy,l,s,theta) -> [n,8] corner coordinates.
 * poly2hbb:  utils/rboxs_utils.py:147-165 — [n,8] -> [n,4] (xc, yc, w, h) of the axis-aligned hull.
 * scale_polys: utils/general.py:636-650 — in place: x -= pad_x, y -= pad_y, all /= gain (un-letterbox).
 * gaussian_label: utils/rboxs_utils.py:9-26 — Circular-Smooth-Label rows [n, num_class] from angles in degrees
 *   (fp64, as numpy evaluates them); peak at bin num_class/2 - trunc(num_class/2 - angle). */
int y5obb_rbox2poly_f32(const float* rboxes5, float* polys8, int64_t n, void* stream);
int y5obb_poly2hbb_f32(const float* polys8, float* hbb4, int64_t n, void* stream);
int y5obb_scale_polys_f32(float* polys8, int64_t n, float pad_x, float pad_y, float gain, void* stream);
/* rbox2poly followed by scale_polys for the packed NMS output of a whole batch, as detect.py:129-147 / val.py:226-232 apply
 * them per image: rows7 [B, max_det, 7] (cx, cy, l, s, theta, conf, cls), counts [>= B] int64 valid rows per image,
 * pad_gain3 [B, 3] fp32 (pad_x, pad_y, gain) per image -> polys8 [B, max_det, 8] in source-image pixels.  The same separately
 * rounded fp32 operations as the two calls above, so the result equals calling them in turn; rows >= counts[b] are zero. */
int y5obb_scale_polys_batched_f32(const float* rows7, const int64_t* counts, const float* pad_gain3, int B, int max_det,
                                  float* polys8, void* stream);
/* poly2rbox (utils/rboxs_utils.py:39-81, whose arithmetic is cv2.minAreaRect): [n,8] fp32 corner points ->
 * [n,5] fp64 (cx, cy, long edge, short edge, theta); theta in [-pi/2, pi/2) with pi = 3.141592 (use_pi) or degrees in [0, 180) */
int y5obb_poly2rbox(const float* polys8, double* rbox5, int64_t n, int use_pi, void* stream);
int y5obb_gaussian_label(const double* angle_deg, float* csl_out, int64_t n, int num_class, double sigma,
                         void* stream);

/* ---- training-mode BatchNorm + SiLU (NHWC bf16) ------------------------------------------------
 * Conv.forward = act(bn(conv(x))) in train mode (models/common.py:45-46; BN eps 1e-3, momentum 0.03,
 * utils/torch_utils.py:160-162).  The conv runs raw (act = 0, zero bias) through y5obb_conv_*; then
 *   y5obb_bn_stats      per-channel sum / sum of squares over npix pixels (fp32; deterministic two-stage reduction:
 *                       block partials in `scratch`, added in block order)
 *   y5obb_bn_finalize   scale = gamma / sqrt(var_biased + eps), shift = beta - mean * scale, mean / invstd saved
 *                       for backward, running statistics updated as torch.nn.BatchNorm2d does (unbiased var)
 *   y5obb_bn_silu_apply y = [res +] act(z * scale + shift) into a channel slice, optional 2x nearest copy (W = image
 *                       width in pixels, needed only for the up-sampled copy) */
int64_t y5obb_bn_scratch_floats(int C);  /* scratch (fp32 elements) the two reductions below need for C channels */
int y5obb_bn_stats(const void* z, int64_t z_pix_stride, int64_t npix, int C, float* sum, float* sumsq, float* scratch,
                   int64_t scratch_floats, void* stream);
/* y5obb_bn_stats + y5obb_bn_finalize in two launches (block partials; ordered reduction + finalisation) */
int y5obb_bn_batch_stats(const void* z, int64_t z_pix_stride, int64_t npix, int C, const float* gamma, const float* beta,
                         float eps, float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                         float* mean_out, float* invstd_out, float* scratch, int64_t scratch_floats, void* stream);
int y5obb_bn_finalize(const float* sum, const float* sumsq, int64_t npix, int C, const float* gamma, const float* beta,
                      float eps, float momentum, float* running_mean, float* running_var, float* scale, float* shift,
                      float* mean_out, float* invstd_out, void* stream);
int y5obb_bn_silu_apply(const void* z, int64_t z_pix_stride, int64_t npix, int C, int W, const float* scale,
                        const float* shift, int act, const void* res, int64_t res_pix_stride, void* y,
                        int64_t y_pix_stride, void* y2x, int64_t y2x_pix_stride, void* stream);

/* backward of y = [res +] act(bn(z)): dz (bf16 NHWC) from dy; optional pass-through of dy into the residual branch's
 * gradient (gres, overwritten or accumulated); dgamma / dbeta (fp32, overwritten or accumulated).  sum_du / sum_dux are
 * [C] fp32 scratch. */
int y5obb_bn_silu_bwd(const void* z, int64_t z_pix_stride, const void* dy, int64_t dy_pix_stride, int64_t npix, int C,
                      const float* scale, const float* shift, const float* mean, const float* invstd, int act,
                      float* sum_du, float* sum_dux, void* dz, int64_t dz_pix_stride, void* gres,
                      int64_t gres_pix_stride, int gres_accumulate, float* dgamma, float* dbeta, int param_accumulate,
                      float* scratch, int64_t scratch_floats, void* stream);
/* ---- weight gradient (wgmma GEMM over the pixel axis) ---------------------------------------------
 * dW[tap][co][ci] (fp32, ACCUMULATED with atomics: zero it first) = sum_{b,ho,wo} dz[b,ho,wo,co] * x[b,s*ho+kh-ph,s*wo+kw-pw,ci].
 * Replaces the cuDNN wgrad autograd calls for models/common.py:37-46 under train.py:333.  Operands are the NHWC bf16
 * gradient / activation buffers themselves (channel slices allowed: pix strides in elements, multiples of 8; rows and
 * images dense).  Any map size; zero padding is implicit. */
typedef struct y5obb_wgrad y5obb_wgrad_t;
typedef struct {
  const void* dz;        /* [B][Ho][Wo][dz_pix_stride] bf16, channels [0, Cout) used */
  int64_t dz_pix_stride;
  const void* x;         /* [B][Hi][Wi][x_pix_stride] bf16, channels [0, Cin) used */
  int64_t x_pix_stride;
  int64_t x_row_stride, x_img_stride;  /* elements; 0 = dense (Wi * x_pix_stride, Hi * row).  With explicit strides
                                          x_pix_stride < Cin is allowed: overlapping pixel windows (the stem reads the
                                          3 horizontal taps x 16 space-to-depth channels as one 48-channel pixel) */
  float* dw;             /* fp32; element (tap, co, ci) at dw[tap*dw_tap_stride + co*dw_co_stride + ci*dw_ci_stride] */
  int64_t dw_tap_stride, dw_co_stride, dw_ci_stride;  /* all 0 = dense [KH*KW][Cout][Cin]; (1, Cin*KH*KW, KH*KW) = the
                                                         nn.Conv2d parameter layout [Cout][Cin][KH][KW] */
  int B, Cout, Ho, Wo, Cin, Hi, Wi;
  int KH, KW, stride, pad_h, pad_w;
  int co_group, co_group_pad;  /* Detect: dz channels come in groups of co_group_pad of which the first co_group are
                                  real (padding rows are skipped): dw row = (co / pad) * group + co % pad.  0 = off */
} y5obb_wgrad_desc;
int y5obb_wgrad_create(const y5obb_wgrad_desc* desc, y5obb_wgrad_t** out);
int y5obb_wgrad_run(const y5obb_wgrad_t* w, void* stream);
void y5obb_wgrad_destroy(y5obb_wgrad_t* w);

/* backward helpers of the training graph (NHWC bf16 gradients):
 *   upsample2x_bwd   nn.Upsample(2x nearest) backward: gdst (+)= 2x2 block sums of gsrc
 *   zero_stuff2x     dst[b,2h,2w,:] = src[b,h,w,:] into a pre-zeroed buffer: the dgrad of a stride-2 conv then is a
 *                    stride-1 conv over it with flipped, transposed weights
 *   maxpool5_bwd     one MaxPool2d(5,1,2) backward step of SPPF (models/common.py:190-196) into an fp32 buffer
 *   add_f32_to_bf16  bf16 slice (+)= fp32 dense buffer
 *   detect_grad_pack loss gradient fp32 [B,na,H,W,no] -> bf16 NHWC [B,H,W,na*bn] (the Detect conv's dz) */
int y5obb_upsample2x_bwd(const void* gsrc, int64_t src_pix_stride, void* gdst, int64_t dst_pix_stride, int64_t npix_dst,
                         int C, int W_dst, int accumulate, void* stream);
int y5obb_zero_stuff2x(const void* src, int64_t src_pix_stride, void* dst, int64_t dst_pix_stride, int64_t npix_src, int C,
                       int W_src, void* stream);
int y5obb_maxpool5_bwd(const void* x_in, int64_t in_pix_stride, const float* gout_f32, const void* gout_bf16,
                       int64_t gout_pix_stride, float* gin_f32, int B, int H, int W, int C, void* stream);
int y5obb_add_f32_to_bf16(const float* src, void* dst, int64_t dst_pix_stride, int64_t npix, int C, int accumulate,
                          void* stream);
int y5obb_detect_grad_pack(const float* g, void* out_nhwc, int B, int na, int H, int W, int no, int bn, void* stream);

/* ---- weight re-packing (every optimiser step, train.py:336) ---------------------------------------
 * fp32 nn.Conv2d parameters [Cout][Cin][KH][KW] -> the bf16 operand layouts the conv kernel's TMA descriptors point at,
 * all layers in one launch.  dst is [taps][rows_pad][cols_pad] bf16 (DETECT_BIAS: fp32 [cols_pad]):
 *   FWD           rows = Cout, cols = Cin                         (y5obb_conv_run forward)
 *   DGRAD         rows = Cin,  cols = Cout, taps flipped          (data gradient = conv with transposed weights)
 *   STEM          the 6x6/s2 stem as a 3x1 conv over the 48-channel space-to-depth window (KH=6,KW=6 in; 3 taps out)
 *   DETECT        rows grouped per anchor: group_real real rows padded to group_pad (models/yolo.py:49-65)
 *   DETECT_DGRAD  rows = Cin, cols grouped per anchor
 *   DETECT_BIAS   fp32 bias, grouped per anchor
 *   DGRAD_S2      data gradient of a 3x3 / stride-2 / pad-1 conv for output-pixel parity (ph, pw) = (group_real >> 1,
 *                 group_real & 1): rows = Cin, cols = Cout, (ph ? 2 : 1) x (pw ? 2 : 1) taps; tap t along an axis of parity 1
 *                 is source tap (t == 0 ? 2 : 0), along an axis of parity 0 source tap 1 */
enum { Y5OBB_PACK_FWD = 0, Y5OBB_PACK_DGRAD = 1, Y5OBB_PACK_STEM = 2, Y5OBB_PACK_DETECT = 3, Y5OBB_PACK_DETECT_DGRAD = 4,
       Y5OBB_PACK_DETECT_BIAS = 5, Y5OBB_PACK_DGRAD_S2 = 6 };
typedef struct y5obb_pack_plan y5obb_pack_plan_t;
typedef struct {
  const float* src;
  void* dst;
  int kind, Cout, Cin, KH, KW, rows_pad, cols_pad, group_real, group_pad;
} y5obb_pack_entry;
int y5obb_pack_plan_create(const y5obb_pack_entry* entries, int n, y5obb_pack_plan_t** out);
int y5obb_pack_plan_run(const y5obb_pack_plan_t* plan, void* stream);
void y5obb_pack_plan_destroy(y5obb_pack_plan_t* plan);

/* ---- fused SGD-Nesterov + EMA step -------------------------------------------------------------------------------
 * train.py:148-162,336-342 + utils/torch_utils.py:304-314 over every tensor in one launch.  group 0/1/2 index the per-step
 * learning-rate table (BatchNorm weights / decayed weights / biases); group -1 = EMA only (floating-point buffers);
 * ema may be NULL. */
typedef struct y5obb_sgd_plan y5obb_sgd_plan_t;
typedef struct {
  float* p;          /* parameter (fp32 master weight), updated in place */
  const float* g;    /* gradient */
  float* mom;        /* momentum buffer */
  float* ema;        /* EMA copy of p, or NULL */
  int64_t n;
  float weight_decay;
  int group;
} y5obb_sgd_entry;
int y5obb_sgd_ema_plan_create(const y5obb_sgd_entry* entries, int n, y5obb_sgd_plan_t** out);
int y5obb_sgd_ema_plan_run(const y5obb_sgd_plan_t* plan, const float* lr3, float momentum, float ema_decay, int first_step,
                           void* stream);
void y5obb_sgd_ema_plan_destroy(y5obb_sgd_plan_t* plan);

/* ---- fused Adam + EMA step ---------------------------------------------------------------------------------------------
 * train.py --adam (train.py:157-163): torch.optim.Adam's multi-tensor step (coupled L2 weight decay, amsgrad off) and
 * utils/torch_utils.py:304-314 over every tensor in one launch, each op rounded as ATen's foreach kernels round it.  group
 * 0/1/2 index the per-step step-size table; group -1 = EMA only (floating-point buffers); ema may be NULL.
 * run: step_size3[k] = -lr_k / (1 - beta1^t) and bc2_sqrt = (1 - beta2^t)^0.5, computed in double and rounded to float as
 * torch does; beta1 / beta2 are the doubles of the parameter group (1 - beta1, beta2 and 1 - beta2 are formed in double
 * and rounded to float here, as torch's scalar arguments are).  beta1 and beta2 must lie in [0, 1), bc2_sqrt be > 0. */
typedef struct y5obb_adam_plan y5obb_adam_plan_t;
typedef struct {
  float* p;           /* parameter (fp32 master weight), updated in place */
  const float* g;     /* gradient */
  float* exp_avg;     /* first moment */
  float* exp_avg_sq;  /* second moment */
  float* ema;         /* EMA copy of p, or NULL */
  int64_t n;
  float weight_decay;
  int group;
} y5obb_adam_entry;
int y5obb_adam_ema_plan_create(const y5obb_adam_entry* entries, int n, y5obb_adam_plan_t** out);
int y5obb_adam_ema_plan_run(const y5obb_adam_plan_t* plan, const float* step_size3, double beta1, double beta2,
                            float bc2_sqrt, float eps, float ema_decay, void* stream);
void y5obb_adam_ema_plan_destroy(y5obb_adam_plan_t* plan);

/* ---- tile-merge polygon NMS of the DOTA devkit (CPU form, double precision) ---------------------------------------
 * DOTA_devkit/ResultMerge_multi_process.py:62-123 py_cpu_nms_poly_fast over DOTA_devkit/polyiou.cpp:106-128 iou_poly, in
 * double precision without FMA contraction (bit-equal to the reference's g++ build by construction; oracle/poly_ref.py).
 * dets9: [n][9] = x1 y1 x2 y2 x3 y3 x4 y4 score (device).  keep_out: indices in descending score order. */
size_t y5obb_poly_nms_workspace_bytes(int64_t n);
int y5obb_poly_nms_f64(const double* dets9, int64_t n, double thresh, int64_t* keep_out, int64_t* n_keep_out, void* workspace,
                       size_t workspace_bytes, void* stream);
int y5obb_poly_iou_pairs_f64(const double* p8, const double* q8, double* iou_out, int64_t n, void* stream);

/* ---- image files of any size: letterbox straight into the stem input ------------------------------------------------------
 * y5obb_letterbox_s2d_u8 replaces the host front end of detect.py and val.py for a batch of B images of different sizes:
 * utils/datasets.py:217-229 (LoadImages.__next__) and :585-590,662-663,702-720 (LoadImagesAndLabels.__getitem__,
 * load_image_label), i.e. cv2.resize to new_w x new_h, utils/augmentations.py:92-128 letterbox's copyMakeBorder with 114,
 * `transpose((2, 0, 1))[::-1]` and the caller's `/ 255`.
 * src: the images as cv2.imread returns them (uint8 HWC BGR), packed back to back; image b starts at byte src_off.
 * desc_dev: B descriptors followed by the per-image tables, one device buffer of desc_bytes bytes; desc_host: the same bytes
 * in host memory, read before the launch to refuse descriptors that reach outside src, the tables or the Hp x Wp image.
 * Table offsets xtab / ytab count 32-bit words from the start of the buffer.
 *   Y5OBB_LB_COPY      new size == source size, no resampling.
 *   Y5OBB_LB_LINEAR    cv2.INTER_LINEAR, 8-bit fixed point.  Per destination column two words: the first source column, and the
 *                      coefficient pair saturate_cast<short>((1 - fx) * 2048) | saturate_cast<short>(fx * 2048) << 16; rows the same.
 *   Y5OBB_LB_AREA_INT  cv2.INTER_AREA by integer factors kx, ky (and INTER_LINEAR when both are exactly 2, which OpenCV
 *                      resamples as INTER_AREA): (sum + 2) >> 2 for 2x2, else round-half-even of (float)sum * inv_area.
 *   Y5OBB_LB_AREA      cv2.INTER_AREA by a fractional factor, shrinking.  Per axis n + 1 first-tap indices, then per tap two
 *                      words (source index, fp32 weight), in OpenCV's table order.
 * Output: y5obb_stem_s2d_u8's layout [B, Hp/2, Wp/2 + 2*pad_cols, 16] bf16; pixel (y, x) is 114 outside
 * [top, top + new_h) x [left, left + new_w), else the resampled source pixel in RGB order.  The pad_cols columns are not
 * written.  The resampled bytes equal the installed OpenCV's bit for bit (oracle/letterbox_ref.py restates them). */
enum { Y5OBB_LB_COPY = 0, Y5OBB_LB_LINEAR = 1, Y5OBB_LB_AREA_INT = 2, Y5OBB_LB_AREA = 3 };
typedef struct {
  int64_t src_off;           /* byte offset of the image in src */
  int32_t h0, w0;            /* source size */
  int32_t new_h, new_w;      /* resampled size */
  int32_t top, left;         /* where the resampled image starts in the Hp x Wp letterboxed image */
  int32_t mode;              /* Y5OBB_LB_* */
  int32_t kx, ky;            /* Y5OBB_LB_AREA_INT: the block */
  float inv_area;            /* Y5OBB_LB_AREA_INT: 1.f / (kx * ky) */
  int32_t xtab, ytab;        /* word offsets of the column / row table */
  int32_t reserved[2];
} y5obb_letterbox_desc;      /* 64 bytes */
int y5obb_letterbox_s2d_u8(const uint8_t* src, int64_t src_bytes, const void* desc_dev, const y5obb_letterbox_desc* desc_host,
                           int64_t desc_bytes, int B, int Hp, int Wp, void* out_nhwc16, int pad_cols, void* stream);

/* ---- whole-scene inference: tile input and tile-merge (DOTA scenes larger than one tile) --------------------------------
 * The reference's route (README.md:24-26): DOTA_devkit/ImgSplit_multi_process.py:226-273 cuts the scene into subsize^2 tiles
 * (zero padding beyond the scene), val.py --save-json detects each one letterboxed to size^2 (114 border, utils/augmentations.py:
 * 92-128; pad=0.5 rect batching), tools/TestJson2VocClassTxt.py and DOTA_devkit/ResultMerge_multi_process.py:62-236 shift the
 * polygons into the scene and run py_cpu_nms_poly_fast per (scene, class).
 *
 * y5obb_scene_tiles_s2d_u8: scene_hwc [H, W, 3] uint8 BGR (as cv2.imread returns it; 64-bit addressing), origins2 [n_tiles, 2]
 * int32 (left, up) -> the stem input of the n_tiles tiles in y5obb_stem_s2d_u8's layout [n_tiles, size/2, size/2 + 2*pad_cols, 16]:
 * tile pixel (y, x) of the size^2 letterboxed tile is 114 outside [border, border + subsize)^2, else scene pixel
 * (up + y - border, left + x - border) in RGB order, or 0 beyond the scene.  The pad_cols columns are not written. */
int y5obb_scene_tiles_s2d_u8(const uint8_t* scene_hwc, int64_t H, int64_t W, const int32_t* origins2, int n_tiles, int subsize,
                             int size, int border, void* out_nhwc16, int pad_cols, void* stream);
/* y5obb_scene_merge_f64: rows7 [n_tiles, max_det, 7] + counts [n_tiles] = the packed output of y5obb_nms_obb_f32 for the tiles
 * (cx, cy, l, s, theta, conf, cls; counts[t] valid rows), origins2 as above -> out10 [K, 10] fp64 rows (class, score, x1 y1 ...
 * x4 y4), per class (ascending) in keep order, *n_out = K (out10 holds n_tiles * max_det rows).  Per row, as the reference's
 * chain computes it: rbox2poly (fp32), scale_polys (x - pad) / gain (fp32), Python round(x, 1) and round(conf, 5) of the fp32
 * values, x + left / y + up in fp64; then per class py_cpu_nms_poly_fast at `thresh` over the candidates sorted by descending
 * rounded score (ties: lower tile * max_det + row first).  Rows of a class outside [0, nc) are ignored.
 * SYNCHRONOUS once: the per-class candidate counts are copied to class_cands_host [nc] (host memory) and the stream is
 * synchronised, because they size the dense suppression masks that follow in the workspace.  Returns Y5OBB_EINVAL when a class
 * has more than Y5OBB_SCENE_MAX_CLASS_CANDIDATES candidates (its dense mask would exceed 512 MiB), and Y5OBB_EWORKSPACE when
 * y5obb_scene_merge_workspace_bytes(n_tiles, max_det, nc, class_cands_host) exceeds workspace_bytes (class_cands_host is
 * filled in both cases; call again with a larger workspace).  With class_cands_host = NULL the query returns the part of the
 * workspace needed before the counts are known. */
#define Y5OBB_SCENE_MAX_CLASS_CANDIDATES 65536
size_t y5obb_scene_merge_workspace_bytes(int64_t n_tiles, int max_det, int nc, const int64_t* class_cands_host);
int y5obb_scene_merge_f64(const float* rows7, const int64_t* counts, const int32_t* origins2, int64_t n_tiles, int max_det,
                          int nc, float pad, float gain, double thresh, double* out10, int64_t* n_out, int64_t* class_cands_host,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---- DOTA Task1 evaluation (OBB mAP of the reference's README) ---------------------------------------------------------
 * y5obb_dota_eval_f64: DOTA_devkit/dota_evaluation_task1.py:88-249 voc_eval + :54-85 voc_ap for every class at once.
 * det10 [n_det, 10] fp64 = (class, score, x1 y1 ... x4 y4) with det_img [n_det] the image index (the layout of
 * SceneDetections.rows); gt10 [n_gt, 10] fp64 = (class, difficult, x1 y1 ... x4 y4) with gt_img [n_gt], difficult non-zero =
 * difficult.  Per class: detections in descending score (ties: lower input index first), each compared with the GTs of its
 * (image, class) in input order through the axis-aligned pre-filter (+1 pixel convention on the intersection and the
 * union) and iou_poly(GT, det); TP / FP / ignored as voc_eval's R['det'] loop decides them; rec = tp / npos,
 * prec = tp / max(tp + fp, DBL_EPSILON); ap by the VOC07 11-point metric (use_07_metric != 0) or the continuous one, with
 * numpy's pairwise summation.  Outputs (device): class_off [nc + 1] (class c's curve is rec / prec [class_off[c],
 * class_off[c + 1])), rec / prec [n_det], ap [nc], npos [nc] (non-difficult GTs), status [1]: 0, or Y5OBB_EINVAL when a row's
 * class is not an integer in [0, nc) or its image is outside [0, n_images) (such rows are left out; the outputs are then
 * not meaningful).  Asynchronous: no host read, no synchronisation.  Returns Y5OBB_EINVAL for negative sizes, nc <= 0 or
 * null pointers, Y5OBB_EWORKSPACE when ws_bytes < y5obb_dota_eval_workspace_bytes(n_det, n_gt, n_images, nc). */
size_t y5obb_dota_eval_workspace_bytes(int64_t n_det, int64_t n_gt, int n_images, int nc);
int y5obb_dota_eval_f64(const int32_t* det_img, const double* det10, int64_t n_det, const int32_t* gt_img, const double* gt10,
                        int64_t n_gt, int n_images, int nc, double ovthresh, int use_07_metric, int64_t* class_off,
                        double* rec, double* prec, double* ap, int64_t* npos, int32_t* status, void* ws, size_t ws_bytes,
                        void* stream);
/* y5obb_task1_round_f64: rows10 [n, 10] (class, score, 8 coordinates) -> out10 with Python's round(score, 2) and
 * round(x, 1), the values the Task1 text of ResultMerge_multi_process.py mergesingle (:221-236) parses back to
 * (dota_evaluation_task1.py:88-249 reads that text). */
int y5obb_task1_round_f64(const double* rows10, int64_t n, double* out10, void* stream);

/* ---- post-NMS geometry + validation matching (SURVEY 8f rank 3)------------------------------------------------------
 * One launch per batch for val.py:226-250 + process_batch (val.py:69-92): detections pred7 [batch, max_det, 7] (the packed
 * output of y5obb_nms_obb_f32, counts[b] valid rows) -> native-space polygons polyn8 [batch, max_det, 8] (rbox2poly +
 * scale_polys) and boxes hbbn4 [batch, max_det, 4] (poly2hbb + xywh2xyxy) (either may be NULL), and correct
 * [batch, max_det, niou] (uint8) against labels7 [n_labels, 7] = (image, cls, cx, cy, l, s, theta) in network-input pixels.
 * scale5 [batch, 5] = (gain, pad_x, pad_y, raw_h, raw_w) per image (shapes[si] of val.py:213).  *overflow_flag is set when an
 * image carries more than 1536 labels (the surplus is ignored). */
int y5obb_val_match_f32(const float* pred7, const int64_t* counts, int batch, int max_det, const float* labels7, int n_labels,
                        const float* scale5, const float* iouv, int niou, uint8_t* correct, float* polyn8, float* hbbn4,
                        int* overflow_flag, void* stream);

/* ---- validation metrics: val.py:209-276 stats + utils/metrics.py:21-114 ap_per_class (plot=False) ---------------------
 * y5obb_val_stats_append: one asynchronous launch per batch.  Appends the valid rows of every image b (the first
 * min(counts[b], max_det) rows of pred7 [batch, max_det, 7], including images without labels) as tp [capacity, niou]
 * (correct [batch, max_det, niou] != 0), conf [capacity] fp32, cls [capacity] int32 and key [capacity] =
 * (image_base + b) << 32 | row, at the running row count *n_rows (device), which it advances.  labels [n_labels,
 * label_stride] fp32 = (image, cls, ...): the classes of the rows whose image is an integer in [0, batch) (including images
 * without detections) are added to nt [nc] (int64).  nms_cap >= 0: counts has batch + 1 entries (non_max_suppression_obb's
 * async form) and the batch is appended only when 0 <= counts[batch] <= nms_cap and no count is negative; otherwise nothing
 * is appended and *skip = 1 (else 0), so that the caller re-runs the batch.  flags [3] int32, zero before the first call:
 * flags[0] |= 1 for a detection or label class that is not an integer in [0, nc) (the row's cls is stored as -1), |= 2 for
 * rows past capacity (not stored); flags[1] = 1 once any appended tp is set (val.py:270 stats[0].any()); flags[2] is the
 * launch's block counter.  batch <= 4096. */
int y5obb_val_stats_append(const float* pred7, const int64_t* counts, int batch, int max_det, int64_t nms_cap,
                           const uint8_t* correct, int niou, const float* labels, int64_t n_labels, int label_stride,
                           int64_t image_base, uint8_t* tp, float* conf, int32_t* cls, int64_t* key, int64_t capacity,
                           int64_t* n_rows, int64_t* nt, int nc, int32_t* flags, int32_t* skip, void* stream);
/* y5obb_ap_per_class_f64: ap_per_class over the first min(*n_rows, capacity) rows, bit for bit in fp64.  The row count stays
 * on the device: every pass runs over the whole capacity and rows past the count carry sentinel keys that sort behind every
 * class, so the call needs no host read.  Rows are ordered by descending conf with ties in ascending key (image, row) order:
 * ordered != 0 promises that the rows were appended in key order, otherwise a radix sort by key comes first.  Classes:
 * those with nt > 0, ascending (np.unique(target_cls)); rows of other classes are ignored.  Outputs (device, the first
 * *n_u rows meaningful, the rest zero): ap [nc, niou] (compute_ap: 101-point np.interp of the suffix-max envelope, np.trapz
 * in numpy's summation order), p / r [nc, 1000] (np.interp on px = np.linspace(0, 1, 1000), left = 1 / 0), ap_class [nc]
 * int32 (-1 past *n_u), n_u [1] int32.  A class with labels but no rows gets zeros.  The 101-point interpolation assumes
 * recall <= 1 in every column (no class has more true positives than labels), which y5obb_val_match_f32 guarantees.
 * Requires capacity * niou <= INT_MAX; Y5OBB_EWORKSPACE when ws_bytes < y5obb_ap_per_class_workspace_bytes. */
size_t y5obb_ap_per_class_workspace_bytes(int64_t capacity, int niou, int nc);
int y5obb_ap_per_class_f64(const uint8_t* tp, const float* conf, const int32_t* cls, const int64_t* key, const int64_t* n_rows,
                           int64_t capacity, int ordered, const int64_t* nt, int nc, int niou, double* ap, double* p, double* r,
                           int32_t* ap_class, int32_t* n_u, void* ws, size_t ws_bytes, void* stream);

/* ---- training augmentation (utils/datasets.py:561-672, utils/augmentations.py:48-61, :131-222, :276-281) -------------
 * Replaces LoadImagesAndLabels.__getitem__ (augment=True, rect=False, perspective == 0) + collate_fn for a batch.  The random
 * draws and the matrices stay on the host (yolov5_obb_b200/augment.py plan_sample); a batch is B records of this layout.
 * Placement p = 4 g + i is image i of group g: group 0 is load_mosaic's 2S mosaic (4 placements, canvas 2S) or the
 * letterboxed image (1 placement, canvas S); group 1 is mixup's second mosaic.  A placement puts image img[p] on the canvas
 * rectangle rect[p] = (x1a, y1a, x2a, y2a), canvas = image + pad[p]; its labels move by lpad[p] (fp32 add).  minv[g] is the
 * inverse warpAffine computes from m[g] = M[:2] of random_perspective (fp64, row-major). */
#define Y5OBB_AUG_MAX_PLACE 8
#define Y5OBB_AUG_MOSAIC 1
#define Y5OBB_AUG_MIXUP 2
#define Y5OBB_AUG_HSV 4
#define Y5OBB_AUG_FLIPUD 8
#define Y5OBB_AUG_FLIPLR 16
typedef struct {
  int32_t img[Y5OBB_AUG_MAX_PLACE];
  int32_t rect[4 * Y5OBB_AUG_MAX_PLACE];
  int32_t pad[2 * Y5OBB_AUG_MAX_PLACE];
  float lpad[2 * Y5OBB_AUG_MAX_PLACE];
  double minv[12], m[12];
  double mix_r, mix_1mr;     /* np.random.beta(32, 32) and 1 - r (mixup, Y5OBB_AUG_MIXUP) */
  int32_t n_place[2], canvas[2];
  int32_t flags, reserved;
  uint8_t lut[768];          /* augment_hsv's hue, saturation, value LUTs (Y5OBB_AUG_HSV) */
} y5obb_augment_sample;
/* The dataset: images uint8 HWC BGR in one flat buffer, labels [*, 9] fp32 (cls, poly) in another; meta [n_images][5] int64 =
 * (image byte offset, h, w, first label row, label count).
 * y5obb_augment_check (host pointers): refuses S not a multiple of 32, images over S or outside the buffers, labels
 * outside the label buffer, and records with bad image ids, placement counts, canvases or rectangles outside the canvas or
 * the image.  The launch entries take device copies of meta and recs; a bad id there is skipped, never read.
 * y5obb_augment_images_u8: out [B, 3, S, S] uint8 RGB (utils/datasets.py:662): per pixel the canvas (never materialised)
 *   sampled by cv2.warpAffine's fixed-point INTER_LINEAR with border 114, mixup's fp64 blend truncated, augment_hsv's
 *   COLOR_BGR2HSV / LUT / COLOR_HSV2BGR round trip (OpenCV 4.13's 8-bit arithmetic), flipud, fliplr.
 * y5obb_augment_labels: candidates are every label of every placement in (sample, placement) order; cand_start [B*8 + 1]
 *   is their exclusive prefix per placement (ncand = cand_start[B*8]).  Each goes through + lpad (fp32), load_mosaic's
 *   poly_filter on the 2S canvas (fp32), xy @ M.T (fp64), poly_filter on S, the cast to fp32, the flips (S - y - 1 in fp32),
 *   poly2rbox and labels_mask (:644-646, quirks included); survivors are compacted in order into rows [nt, tcols]:
 *   tcols = 7 + nc_theta -> (image, cls, cx, cy, l, s, theta, CSL row of sigma csl_radius); tcols == 8 -> column 7 is
 *   int(nc_theta / 2 - angle) (the loss's compact layout).  *nt (device) receives the count; rows needs ncand * tcols floats. */
int y5obb_augment_check(const int64_t* meta, int n_images, int64_t images_bytes, int64_t n_labels,
                        const y5obb_augment_sample* recs, int B, int S);
int y5obb_augment_images_u8(const uint8_t* images, const int64_t* meta, int n_images, const y5obb_augment_sample* recs,
                            int B, int S, uint8_t* out, void* stream);
size_t y5obb_augment_labels_workspace_bytes(int64_t ncand);
int y5obb_augment_labels(const float* labels, const int64_t* meta, int n_images, const y5obb_augment_sample* recs,
                         const int64_t* cand_start, int B, int64_t ncand, int S, int nc_theta, double csl_radius, int tcols,
                         float* rows, int64_t* nt, void* workspace, size_t workspace_bytes, void* stream);

/* ---- float polygon NMS / rotated-box overlaps (rows A14, B4)---------------------------------------------------------
 * Device-pointer forms of  utils/nms_rotated/src/nms_rotated_ext.cpp:42-55 nms_poly -> src/poly_nms_cuda.cu:144-261 (K2),
 * DOTA_devkit/poly_nms_gpu/poly_nms_kernel.cu:214-329 (K3) and poly_overlaps_kernel.cu:283-427 (K4); the float polygon IoU
 * restates the reference's expression by expression (union == 0 -> (inter + 1) / (union + 1)).
 * dets9 [n][9] = x1 y1 x2 y2 x3 y3 x4 y4 score.  presorted = 0: polygons are processed by descending score (stable: ties ->
 * lower index), as nms_poly / poly_gpu_nms do before calling the kernel; 1: in the caller's order (the _poly_nms contract).
 * keep_out: indices into dets9 in processing order.  overlaps [n][k] = IoU(boxes5[i], query5[j]), boxes (cx, cy, w, h, angle). */
size_t y5obb_poly_nms_f32_workspace_bytes(int64_t n);
int y5obb_poly_nms_f32(const float* dets9, int64_t n, float iou_thr, int presorted, int64_t* keep_out, int64_t* n_keep_out,
                       void* workspace, size_t workspace_bytes, void* stream);
int y5obb_poly_overlaps_f32(const float* boxes5, const float* query5, int64_t n, int64_t k, float* overlaps, void* stream);
int y5obb_poly_iou_pairs_f32(const float* p8, const float* q8, float* iou_out, int64_t n, void* stream);
/* The devkit's own C ABI (B4): host pointers in and out, synchronous, default stream, CUDA errors printed to stdout - the
 * signatures of DOTA_devkit/poly_nms_gpu/poly_nms.hpp:9-10 and poly_overlaps.hpp:1.  The library also exports them under the
 * reference's C++ names `_poly_nms` / `_overlaps` (include/y5obb_devkit.hpp), which is what the devkit's .pyx files link. */
void y5obb_devkit_poly_nms(int* keep_out_host, int* num_out_host, const float* polys_host, int polys_num, int polys_dim,
                           float nms_overlap_thresh, int device_id);
void y5obb_devkit_overlaps(float* overlaps_host, const float* boxes_host, const float* query_boxes_host, int n, int k,
                           int device_id);

#ifdef __cplusplus
}
#endif
#endif /* Y5OBB_H_ */
