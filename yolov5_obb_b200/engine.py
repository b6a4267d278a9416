"""Inference plan: turns a yolo.Model into a fixed sequence of sm_90a kernel launches.

Layout decisions (all NHWC bf16, or fp16 for a model whose parameters are fp16, see plan_dtype):
  * every tensor is a channel slice of some buffer; a producer whose output feeds a Concat
    (models/common.py:267-274) stores directly at its channel offset in the concat buffer;
  * nn.Upsample(2x nearest) is a second store of the producing conv's epilogue (out2x);
  * C3 (models/common.py:126-138): cv1 and cv2 share the input, so they run as ONE GEMM with
    concatenated output channels [cv1 | cv2] written into the block's concat buffer; the Bottleneck
    chain then updates channels [0, c_) in place (1x1 -> tmp, 3x3 + residual -> back), cv3 reads the
    whole buffer;
  * SPPF (:181-196): cv1 -> channels [0,c_) of a 4c_ buffer, one pooling kernel fills the rest;
  * the stem Conv(3, c, 6, 2, 2) runs as a 3x3 conv over a 2x2 space-to-depth copy of the image;
  * Detect (models/yolo.py:49-81): one GEMM per level whose epilogue permutes, applies sigmoid and the
    grid/anchor decode and writes fp32 rows of the final [B, A, no] tensor.
BatchNorm is folded into the conv weights exactly as utils/torch_utils.py:192-212 (fuse_conv_and_bn).
fp16 plans are the reference's half inference (val.py --half, detect.py --half): the fused weights and biases are rounded to
fp16, activations are fp16, and the Detect epilogue computes models/yolo.py:63-77 on a half tensor (Y5OBB_CONV_F16).
"""
import ctypes
import math
import os
from typing import List, Optional

import numpy as np
import torch

from . import _lib
from .conv import Conv as ConvOp, Slice, pack_weights, MODE_DETECT, F16
from .general import require_nc
from .layout import _is, route, shapes, sources, stem_weight, stem_window
from . import yolo as Y


def fold_bn(conv: torch.nn.Conv2d, bn: Optional[torch.nn.BatchNorm2d]):
    """W' = diag(gamma / sqrt(var + eps)) W ; b' = beta - gamma * mean / sqrt(var + eps)  (+ conv bias).
    Host-side plan building: the arithmetic runs on CPU copies of the parameters (one D2H copy per tensor, no device
    kernels), the packed bf16 operands are uploaded once by the caller."""
    w = conv.weight.detach().float().cpu()
    b = conv.bias.detach().float().cpu() if conv.bias is not None else torch.zeros(w.shape[0])
    if bn is None:
        return w, b
    scale = bn.weight.detach().float().cpu() / torch.sqrt(bn.running_var.detach().float().cpu() + bn.eps)
    return w * scale.view(-1, 1, 1, 1), (b - bn.running_mean.detach().float().cpu()) * scale + bn.bias.detach().float().cpu()


def _conv_params(m):
    return fold_bn(m.conv, getattr(m, "bn", None))


def plan_dtype(model) -> torch.dtype:
    """The element type of a model's inference plans: fp16 when its parameters are fp16 (`model.half()`: a half model runs
    half, as in torch), bf16 otherwise.  Plans of the two kinds are separate (yolo.Model keys them by it)."""
    dts = {p.dtype for p in model.parameters()}
    if torch.float16 in dts and len(dts) > 1:
        raise RuntimeError(f"the model mixes parameter dtypes {sorted(str(d) for d in dts)}: call .half() or .float() on it")
    return torch.float16 if dts == {torch.float16} else torch.bfloat16


def stage_input(x: torch.Tensor, x_s2d: torch.Tensor) -> None:
    """The stem layout pass: x [B, 3, H, W] contiguous fp32 in [0, 1] or uint8 (the caller-side `/ 255` is folded in) ->
    the space-to-depth stem input x_s2d (bf16, or fp16 for an fp16 plan), on the current stream."""
    B, _, H, W = x.shape
    L, st = _lib.lib(), _lib.stream_ptr(x_s2d.device)
    sfx = "_f16" if x_s2d.dtype == torch.float16 else ""
    name = ("y5obb_stem_s2d_u8" if x.dtype == torch.uint8 else "y5obb_stem_s2d") + sfx
    _lib.check(getattr(L, name)(x.data_ptr(), x_s2d.data_ptr(), B, H, W, 1, st), name)


class InferenceEngine:
    def __init__(self, model: "Y.Model", B: int, H: int, W: int, device, conv_flags: int = 0, compact_detect: bool = False,
                 det_out: Optional[torch.Tensor] = None, det_row_base: int = 0, levels=None, descale=None,
                 x_s2d: Optional[torch.Tensor] = None):
        """The keyword options let several plans write one output (TTAPlan, EnsemblePlan); their defaults give the plain plan:
        det_out       an external [B, rows_per_image, no | rec_w] fp32 tensor the Detect epilogue writes into, from row
                      `det_row_base` of every image on (default: an engine-owned tensor holding exactly this plan's rows);
        levels        the Detect levels to emit (default all).  Ops whose outputs reach no kept level are not emitted;
        descale       (inv_scale, flip_w): the Detect epilogue de-scales x y w h and de-flips x (y5obb_conv_desc.det_descale);
        x_s2d         an external stem input [B, H/2, W/2 + 2, 16] of the plan's dtype whose two padding columns are zero
                      (default: an engine-owned zeroed one).  Plans that share it read one staged image (EnsemblePlan).
        The plan's element type is plan_dtype(model): an fp16 plan's eval rows (`pred` without compact_detect) are fp16,
        its compact records fp32 holding fp16 values."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("InferenceEngine needs a CUDA device (sm_90a); there is no CPU path")
        det = model.model[-1]
        require_nc(det.nc, "InferenceEngine")
        smax = int(max(model.stride))
        if H % smax or W % smax:
            raise RuntimeError(f"image size {H}x{W} must be a multiple of the max stride {smax}")
        self.device, self.B, self.H, self.W = device, B, H, W
        self.dtype = plan_dtype(model)
        self.half = self.dtype == torch.float16
        if self.half:
            conv_flags |= F16
        self.ops = []          # (callable taking stream ptr)
        self._calls, self._graph = 0, None
        self._use_graph = os.environ.get("Y5OBB_NO_GRAPH", "0") != "1"
        self.convs: List[ConvOp] = []
        self.keep = []         # buffers
        self.flops = 0.0
        self.hbm_bytes = 0.0
        L = _lib.lib()
        layers = list(model.model)
        n = len(layers)
        ch, hw = shapes(layers, H, W)

        # ---- liveness: backwards from the inputs of the kept Detect levels (a pruned level's head is not emitted)
        self.levels = tuple(range(det.nl)) if levels is None else tuple(sorted(set(int(l) for l in levels)))
        if not self.levels or not all(0 <= l < det.nl for l in self.levels):
            raise RuntimeError(f"Detect levels {levels} are not a non-empty subset of 0..{det.nl - 1}")
        live = [False] * n
        need = {det.f[l] for l in self.levels}
        for m in reversed(layers[:-1]):
            if m.i in need:
                live[m.i] = True
                need.update(sources(m))

        arena = {"buf": None, "used": 0}

        def new(h, w, c):
            # zeros, once: the pixel-pair view of stride-2 convs may read channels of a buffer before their
            # producer ran (they meet zero weights, but must be finite).  Carved from a few large zeroed chunks
            # (one fill each) instead of one allocation + fill per tensor.
            n = B * h * w * c
            n_al = (n + 127) // 128 * 128   # 256-byte aligned starts (TMA wants 16)
            if arena["buf"] is None or arena["used"] + n_al > arena["buf"].numel():
                arena["buf"] = torch.zeros(max(n_al, 128 << 20), dtype=self.dtype, device=device)
                arena["used"] = 0
                self.keep.append(arena["buf"])
            t = arena["buf"][arena["used"]:arena["used"] + n].view(B, h, w, c)
            arena["used"] += n_al
            return t

        out, up_of = route(layers, ch, hw, new)
        self.out_slices = out   # per top-level layer: where its output lives (tests read them for teacher-forced parity)

        def add_conv(x, w, b, k, s, p, act, dst: Optional[Slice] = None, res=None, out2x=None, detd=None):
            if self.half:   # model.half() rounds the fused bias too (attempt_load fuses in fp32 first); it stays an fp32 array
                b = b.to(torch.float16).float()
            wp, bp = pack_weights(w.cpu(), b.cpu(), MODE_DETECT if detd else 0, detd["no"] if detd else 0,
                                  self.dtype)   # packed on the host
            if act and not detd:
                bp = bp * 0.5   # the SiLU epilogue wants 0.5 * bias (Y5OBB_CONV_BIAS_HALVED)
            op = ConvOp(x, wp.to(device), bp.to(device), w.shape[0], k, s, p, act, out=dst, res=res, out2x=out2x, det=detd,
                        flags=conv_flags, bias_prehalved=True)
            self.convs.append(op)
            info = op.info()
            self.flops += info["flops"]
            self.hbm_bytes += info["hbm_bytes"]
            h = op._h
            self.ops.append(lambda st, h=h: L.y5obb_conv_run(h, st))
            self.op_layers.append(cur[0])

        # ---- pass 3: emit ops
        # space-to-depth image with one zero pixel of padding left and right of every row: the stem's three
        # horizontal taps are then 48 CONTIGUOUS channels of an overlapping-window view (pixel stride 16)
        s2d_shape = (B, H // 2, W // 2 + 2, 16)
        if x_s2d is None:
            self.x_s2d = torch.zeros(s2d_shape, dtype=self.dtype, device=device)
        else:
            _lib.require_cuda(x_s2d, "x_s2d")
            if (tuple(x_s2d.shape) != s2d_shape or x_s2d.dtype != self.dtype or not x_s2d.is_contiguous()
                    or x_s2d.device != device):
                raise RuntimeError(f"x_s2d must be a contiguous {self.dtype} {list(s2d_shape)} tensor on {device}, got "
                                   f"{tuple(x_s2d.shape)} {x_s2d.dtype} on {x_s2d.device}")
            self.x_s2d = x_s2d
        self.keep.append(self.x_s2d)
        self.op_layers = []    # per op: the top-level layer index it belongs to, ("Detect", level) for the head convs
        cur = [None]
        for m in layers:
            i = m.i
            if _is(m, "Detect"):
                break
            if not live[i]:
                continue
            cur[0] = i
            fs = sources(m)
            if _is(m, "Conv"):
                w, b = _conv_params(m)
                k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
                act = isinstance(m.act, torch.nn.SiLU)
                if i == 0:
                    if (k, s, p, w.shape[1]) != (6, 2, 2, 3):
                        raise RuntimeError("layer 0 must be the v6.0 stem Conv(3, c, 6, 2, 2)")
                    add_conv(stem_window(self.x_s2d), stem_weight(w), b, (3, 1), 1, (1, 0), act, out[i])
                else:
                    add_conv(out[fs[0]], w, b, k, s, p, act, out[i], out2x=up_of.get(i))
            elif _is(m, "C3"):
                x = out[fs[0]]
                c_ = m.cv1.conv.out_channels
                cat = Slice.full(new(hw[i][0], hw[i][1], 2 * c_))
                tmp = Slice.full(new(hw[i][0], hw[i][1], c_))
                w1, b1 = _conv_params(m.cv1)
                w2, b2 = _conv_params(m.cv2)
                add_conv(x, torch.cat([w1, w2], 0), torch.cat([b1, b2], 0), 1, 1, 0, True, cat)
                chain = Slice(cat.buf, 0, c_)
                for bt in m.m:
                    wa, ba = _conv_params(bt.cv1)
                    wb, bb = _conv_params(bt.cv2)
                    add_conv(chain, wa, ba, 1, 1, 0, True, tmp)
                    add_conv(tmp, wb, bb, 3, 1, 1, True, chain, res=chain if bt.add else None)
                w3, b3 = _conv_params(m.cv3)
                add_conv(cat, w3, b3, 1, 1, 0, True, out[i])
            elif _is(m, "SPPF"):
                x = out[fs[0]]
                # the pooling kernel is the 5x5 / stride 1 / pad 2 window of every shipped yaml (common.py:183-196); the mirror
                # keeps `k`, the reference's module keeps the nn.MaxPool2d as `m`
                pk = getattr(m, "k", None)
                if pk is None and hasattr(m, "m"):
                    pk = m.m.kernel_size if isinstance(m.m.kernel_size, int) else m.m.kernel_size[0]
                if pk != 5:
                    raise RuntimeError(f"SPPF with a {pk}x{pk} pooling window is not planned (the kernel is 5x5)")
                c_ = m.cv1.conv.out_channels
                cat4 = new(hw[i][0], hw[i][1], 4 * c_)
                w1, b1 = _conv_params(m.cv1)
                add_conv(x, w1, b1, 1, 1, 0, True, Slice(cat4, 0, c_))
                hh, ww = hw[i]
                ptr, ps = cat4.data_ptr(), cat4.shape[3]
                pool = L.y5obb_sppf_pool_f16 if self.half else L.y5obb_sppf_pool
                self.ops.append(lambda st, ptr=ptr, ps=ps, hh=hh, ww=ww, c_=c_: pool(ptr, ps, B, hh, ww, c_, st))
                self.op_layers.append(i)
                self.hbm_bytes += 2.0 * B * hh * ww * c_ * 4
                w2, b2 = _conv_params(m.cv2)
                add_conv(Slice.full(cat4), w2, b2, 1, 1, 0, True, out[i])
            # Concat / Upsample emit nothing

        # ---- Detect
        self.no, self.na = det.no, det.na
        rows = [det.na * hw[det.f[l]][0] * hw[det.f[l]][1] for l in self.levels]
        self.rows_total = sum(rows)
        # compact_detect: the Detect epilogue writes (cx, cy, w, h, obj, cls[nc], theta index) records - all that
        # non_max_suppression_obb reads of a row - instead of the [B, A, no] tensor (96 B instead of 800 B per anchor row)
        self.compact_detect = bool(compact_detect)
        self.rec_w = ((det.nc + 6) + 3) // 4 * 4
        self.nc = det.nc
        width = self.rec_w if compact_detect else det.no
        self.pred_dtype = torch.float16 if self.half and not compact_detect else torch.float32
        if det_out is None:
            if det_row_base:
                raise RuntimeError("det_row_base needs an external det_out")
            self.pred = torch.empty((B, self.rows_total, width), dtype=self.pred_dtype, device=device)
        else:
            _lib.require_cuda(det_out, "det_out")
            if (det_out.dtype != self.pred_dtype or not det_out.is_contiguous() or det_out.dim() != 3 or det_out.shape[0] != B
                    or det_out.shape[2] != width or det_out.device != device or det_row_base < 0
                    or det_row_base + self.rows_total > det_out.shape[1]):
                raise RuntimeError(f"det_out must be a contiguous {self.pred_dtype} [{B}, >= {det_row_base + self.rows_total}, "
                                   f"{width}] "
                                   f"tensor on {device}, got {tuple(det_out.shape)} {det_out.dtype}")
            self.pred = det_out
        row_off = int(det_row_base)
        # what ComputeLoss.head_items needs to check the Detect it is given and to recompute the head's logits
        self.det_nl = det.nl
        self.det_anchors = [float(v) for v in det.anchors.detach().float().cpu().flatten().tolist()]
        self.det_strides = [float(s) for s in det.stride]
        self._head = []
        for l, f in ((l, det.f[l]) for l in self.levels):
            cur[0] = ("Detect", l)
            mi = det.m[l]
            stride = float(det.stride[l])
            anchors_px = (det.anchors[l].detach().float().cpu() * stride).flatten().tolist()
            w, b = mi.weight.detach().float().cpu(), mi.bias.detach().float().cpu()
            add_conv(out[f], w, b, 1, 1, 0, False,
                     detd=dict(out=self.pred, rows_per_image=self.pred.shape[1], row_off=row_off, no=det.no,
                               decode=2 if compact_detect else True,
                               stride=stride, anchors_px=anchors_px, descale=descale))
            # the GEMM's operands: pack_weights rounds the same fp32 values to the plan's dtype, the bias stays fp32
            self._head.append((out[f], w.reshape(w.shape[0], -1).to(self.dtype).to(device), b.to(device)))
            row_off += det.na * hw[f][0] * hw[f][1]
        self.hbm_bytes += (self.pred.element_size() * B * self.rows_total * det.no + 4.0 * B * 3 * H * W
                           + 2.0 * self.x_s2d.numel())
        self.n_launches = len(self.ops) + 1

    def head_inputs(self):
        """Per emitted Detect level: (input Slice, weight [na * no, C] of the plan's dtype, fp32 bias [na * no]) - the Detect
        GEMM's operands.
        The input holds the features of the last forward until the next one, as `pred` does."""
        return list(self._head)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x: [B,3,H,W] fp32 in [0,1] (or uint8 0..255) on this engine's device -> pred [B, A, no] fp32, fp16 for an fp16
        plan (engine-owned buffer, overwritten by the next call).  A half image is widened exactly and rounded back."""
        _lib.require_cuda(x, "x")
        if tuple(x.shape) != (self.B, 3, self.H, self.W):
            raise RuntimeError(f"engine was planned for {(self.B, 3, self.H, self.W)}, got {tuple(x.shape)}")
        with torch.cuda.device(self.device):
            stage_input(x.contiguous() if x.dtype == torch.uint8 else x.contiguous().float(), self.x_s2d)
            return self._run_layers()

    def forward_s2d(self) -> torch.Tensor:
        """Runs the plan on an `x_s2d` the caller has already filled (y5obb_scene_tiles_s2d_u8 writes the stem input of
        scene tiles there) -> pred (or the compact records), engine-owned as in forward()."""
        with torch.cuda.device(self.device):
            return self._run_layers()

    def _run_layers(self) -> torch.Tensor:
        # the layer sequence is fixed (same buffers every call): from the third call on it is replayed as one CUDA
        # graph - the layout pass stays outside because it reads the caller's tensor (Y5OBB_NO_GRAPH=1 disables)
        self._calls += 1
        if self._use_graph and self._calls > 2:
            if self._graph is None:
                torch.cuda.synchronize(self.device)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    self._run_ops(_lib.stream_ptr(self.device))
                self._graph = g
            self._graph.replay()
        else:
            self._run_ops(_lib.stream_ptr(self.device))
        return self.pred

    def _run_ops(self, st):
        for op in self.ops:
            rc = op(st)
            if rc:
                _lib.check(rc, "engine op")


# ---- test-time augmentation (models/yolo.py:149-209 _forward_augment)
TTA_SCALES = (1, 0.83, 0.67)   # yolo.py:151
TTA_FLIPS = (None, 3, None)    # 3 = left-right (x.flip(3))
TTA_PAD = 0.447                # scale_img's F.pad value (utils/torch_utils.py:249)


def tta_geometry(H: int, W: int, gs: int = 32, nl: int = 3, na: int = 3, strides=(8, 16, 32)):
    """Host geometry of _forward_augment for an H x W input (multiples of gs): per branch the scale and flip, scale_img's
    resampled size (h, w) and padded size (Hp, Wp) in its own Python float arithmetic, the Detect levels _clip_augmented keeps
    (the first branch loses its last level, the last branch its first one: for gs-multiple shapes its `shape[1] // g * 4**k`
    row counts are exactly those levels), the branch's rows per image, its first row in the concatenated output, and the
    de-scale constants (the fp32 reciprocal of the fp32 scale, ATen's `/= s` on CUDA; the de-flip width, 0 = none).
    Returns (branches, rows_per_image)."""
    if H % gs or W % gs or H <= 0 or W <= 0:
        raise RuntimeError(f"test-time augmentation needs an image size that is a multiple of {gs}, got {H}x{W}")
    branches, row = [], 0
    last = len(TTA_SCALES) - 1
    for k, (s, fl) in enumerate(zip(TTA_SCALES, TTA_FLIPS)):
        if s == 1.0:
            h, w, Hp, Wp = H, W, H, W
        else:
            h, w = int(H * s), int(W * s)
            Hp, Wp = (math.ceil(v * s / gs) * gs for v in (H, W))
        levels = list(range(nl))
        if k == 0:
            levels = levels[:-1]
        if k == last:
            levels = levels[1:]
        level_rows = [na * (Hp // st) * (Wp // st) for st in strides]
        rows = sum(level_rows[l] for l in levels)
        branches.append(dict(scale=s, flip=fl, h=h, w=w, Hp=Hp, Wp=Wp, levels=tuple(levels), level_rows=level_rows,
                             row_off=row, rows=rows, inv_scale=float(np.float32(1.0) / np.float32(s)),
                             flip_w=float(W) if fl == 3 else 0.0))
        row += rows
    return branches, row


class TTAPlan:
    """_forward_augment on the device: three InferenceEngines (one per scale) whose Detect epilogues de-scale their rows and
    write them into one shared [B, rows_total, no] (or compact-record) tensor at the branch's row offset, so that the
    torch.cat of the clipped branches is never formed.  Branch 0 runs the plain stem layout pass; branches 1 and 2 resample
    the input into their stem buffer (y5obb_scale_img_s2d) and run forward_s2d().  Every plan skips the ops that feed only the
    Detect level _clip_augmented drops.  All work is on the current stream; each engine replays its own CUDA graph.
    As InferenceEngine, the plan can write into an external det_out from row det_row_base on, and `stems` (one entry per
    branch, None = engine-owned) gives its engines external stem inputs, so that several plans share them (EnsemblePlan)."""

    def __init__(self, model: "Y.Model", B: int, H: int, W: int, device, compact_detect: bool = False, conv_flags: int = 0,
                 det_out: Optional[torch.Tensor] = None, det_row_base: int = 0, stems=None):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("TTAPlan needs a CUDA device (sm_90a); there is no CPU path")
        det = model.model[-1]
        require_nc(det.nc, "TTAPlan")
        self.branches, self.rows_total = tta_geometry(H, W, int(max(model.stride)), det.nl, det.na,
                                                      [int(s) for s in det.stride])
        self.device, self.B, self.H, self.W = device, B, H, W
        self.nc, self.no = det.nc, det.no
        self.rec_w = ((det.nc + 6) + 3) // 4 * 4
        self.compact_detect = bool(compact_detect)
        self.dtype = plan_dtype(model)
        self.half = self.dtype == torch.float16
        if det_out is None:
            if det_row_base:
                raise RuntimeError("det_row_base needs an external det_out")
            det_out = torch.empty((B, self.rows_total, self.rec_w if compact_detect else det.no),
                                  dtype=torch.float16 if self.half and not compact_detect else torch.float32, device=device)
        self.pred = det_out
        stems = [None] * len(self.branches) if stems is None else list(stems)
        if len(stems) != len(self.branches):
            raise RuntimeError(f"stems needs one entry per branch ({len(self.branches)}), got {len(stems)}")
        self.engines = [InferenceEngine(model, B, g["Hp"], g["Wp"], device, conv_flags, compact_detect, det_out=self.pred,
                                        det_row_base=int(det_row_base) + g["row_off"], levels=g["levels"],
                                        descale=None if g["scale"] == 1 else (g["inv_scale"], g["flip_w"]), x_s2d=xs)
                        for g, xs in zip(self.branches, stems)]
        self.flops = sum(e.flops for e in self.engines)

    def resample_bytes(self, k: int, itemsize: int = 4) -> float:
        """Algorithmic bytes of branch k's resample: one read of the input plus the stem-layout output."""
        g = self.branches[k]
        return float(self.B) * (3 * self.H * self.W * itemsize + (g["Hp"] // 2) * (g["Wp"] // 2) * 32)

    def resample(self, x: torch.Tensor, k: int) -> None:
        """scale_img of branch k (k >= 1) into that engine's x_s2d."""
        g, e = self.branches[k], self.engines[k]
        name = ("y5obb_scale_img_s2d_u8" if x.dtype == torch.uint8 else "y5obb_scale_img_s2d") + ("_f16" if self.half else "")
        fn = getattr(_lib.lib(), name)
        _lib.check(fn(x.data_ptr(), e.x_s2d.data_ptr(), self.B, self.H, self.W, g["h"], g["w"], g["Hp"], g["Wp"],
                      1 if g["flip"] == 3 else 0, TTA_PAD, 1, _lib.stream_ptr(self.device)), "y5obb_scale_img_s2d")

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x: [B,3,H,W] fp32 in [0,1] (or uint8 0..255) on this plan's device -> [B, rows_total, no] fp32 (or the compact
        records), plan-owned, overwritten by the next call."""
        _lib.require_cuda(x, "x")
        if tuple(x.shape) != (self.B, 3, self.H, self.W):
            raise RuntimeError(f"TTA plan was built for {(self.B, 3, self.H, self.W)}, got {tuple(x.shape)}")
        x = x.contiguous() if x.dtype == torch.uint8 else x.contiguous().float()
        with torch.cuda.device(self.device):
            self.engines[0].forward(x)
            for k in range(1, len(self.engines)):
                self.resample(x, k)
                self.engines[k].forward_s2d()
        return self.pred


# ---- model ensembles (models/experimental.py:74-87 Ensemble: the members' rows concatenated along dim 1, one NMS after)
def ensemble_layout(models, H: int, W: int, augment: bool = False):
    """Host row layout of an ensemble's output for an H x W input: the members' rows in list order, each member's in its own
    level order - with augment=True its own _forward_augment branches, padded to its OWN largest stride (yolo.py:152), so a
    P5 and a P6 member pad their 0.83 / 0.67 branches to multiples of 32 and 64.  H and W must be multiples of the largest
    stride of all members (DetectMultiBackend sizes images by it).  Returns (per-member first row, rows per image)."""
    models = list(models)
    smax = max(int(max(m.stride)) for m in models)
    if H % smax or W % smax or H <= 0 or W <= 0:
        raise RuntimeError(f"image size {H}x{W} must be a multiple of the ensemble's largest stride {smax}")
    bases, row = [], 0
    for m in models:
        det = m.model[-1]
        strides = [int(s) for s in det.stride]
        if augment:
            rows = tta_geometry(H, W, int(max(m.stride)), det.nl, det.na, strides)[1]
        else:
            rows = sum(det.na * (H // s) * (W // s) for s in strides)
        bases.append(row)
        row += rows
    return bases, row


class EnsemblePlan:
    """Ensemble.forward / forward_augment / detect_records on the device: one plan per member (InferenceEngine, or TTAPlan for
    augment=True) whose Detect epilogues write the member's rows into one shared [B, rows_total, no] (or compact-record)
    tensor from the member's row base on, so the torch.cat of the members' outputs is never formed.  The image is staged
    once (one stem layout pass into `x_s2d`) and every member's stem reads it; with augment=True the scale-1 branches read it
    too, and each resampled branch input is made once per (scale, member gs) and read by every member with that gs.
    `steps` lists what forward runs, in order, as (label, fn(x)): ("stem",), ("resample", branch, gs), ("layers", member,
    branch).  All work is on the current stream; each engine replays its own CUDA graph."""

    def __init__(self, models, B: int, H: int, W: int, device, compact_detect: bool = False, augment: bool = False,
                 conv_flags: int = 0):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("EnsemblePlan needs a CUDA device (sm_90a); there is no CPU path")
        models = list(models)
        if not models:
            raise RuntimeError("an ensemble needs at least one member")
        ncs = sorted({int(m.model[-1].nc) for m in models})
        if len(ncs) != 1:
            raise RuntimeError(f"ensemble members have different class counts {ncs}: their rows cannot be concatenated")
        require_nc(ncs[0], "EnsemblePlan")
        dts = {plan_dtype(m) for m in models}
        if len(dts) != 1:
            raise RuntimeError("ensemble members mix fp16 and fp32 parameters: call .half() or .float() on the ensemble")
        self.dtype = dts.pop()
        self.half = self.dtype == torch.float16
        self.row_bases, self.rows_total = ensemble_layout(models, H, W, augment)
        self.device, self.B, self.H, self.W = device, B, H, W
        self.nc = ncs[0]
        self.no = self.nc + 185
        self.rec_w = ((self.nc + 6) + 3) // 4 * 4
        self.compact_detect, self.augment = bool(compact_detect), bool(augment)
        self.pred = torch.empty((B, self.rows_total, self.rec_w if compact_detect else self.no),
                                dtype=torch.float16 if self.half and not compact_detect else torch.float32, device=device)
        self.x_s2d = torch.zeros((B, H // 2, W // 2 + 2, 16), dtype=self.dtype, device=device)
        self.steps = [(("stem",), lambda x: stage_input(x, self.x_s2d))]
        if not augment:
            self.members = [InferenceEngine(m, B, H, W, device, conv_flags, compact_detect, det_out=self.pred,
                                            det_row_base=base, x_s2d=self.x_s2d)
                            for m, base in zip(models, self.row_bases)]
            for i, e in enumerate(self.members):
                self.steps.append((("layers", i, 0), lambda x, e=e: e.forward_s2d()))
        else:
            gss = [int(max(m.stride)) for m in models]
            stems = {}   # gs -> per branch stem input; branch 0 (scale 1, no padding) is the staged image itself
            for gs in sorted(set(gss)):
                stems[gs] = [self.x_s2d] + [torch.zeros((B, g["Hp"] // 2, g["Wp"] // 2 + 2, 16), dtype=self.dtype,
                                                        device=device) for g in tta_geometry(H, W, gs)[0][1:]]
            self.members = [TTAPlan(m, B, H, W, device, compact_detect, conv_flags, det_out=self.pred, det_row_base=base,
                                    stems=stems[gs]) for m, base, gs in zip(models, self.row_bases, gss)]
            for i, p in enumerate(self.members):
                self.steps.append((("layers", i, 0), lambda x, e=p.engines[0]: e.forward_s2d()))
            for k in range(1, len(TTA_SCALES)):
                for gs in sorted(set(gss)):
                    idx = [i for i, g in enumerate(gss) if g == gs]
                    self.steps.append((("resample", k, gs), lambda x, p=self.members[idx[0]], k=k: p.resample(x, k)))
                    for i in idx:
                        self.steps.append((("layers", i, k), lambda x, e=self.members[i].engines[k]: e.forward_s2d()))
        for p, base in zip(self.members, self.row_bases):
            assert p.pred is self.pred and base + p.rows_total <= self.rows_total
        self.flops = sum(p.flops for p in self.members)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x: [B,3,H,W] fp32 in [0,1] (or uint8 0..255) on this plan's device -> [B, rows_total, no] fp32 (or the compact
        records), plan-owned, overwritten by the next call."""
        _lib.require_cuda(x, "x")
        if tuple(x.shape) != (self.B, 3, self.H, self.W):
            raise RuntimeError(f"ensemble plan was built for {(self.B, 3, self.H, self.W)}, got {tuple(x.shape)}")
        x = x.contiguous() if x.dtype == torch.uint8 else x.contiguous().float()
        with torch.cuda.device(self.device):
            for _, fn in self.steps:
                fn(x)
        return self.pred

    def forward_s2d(self) -> torch.Tensor:
        """Runs every member on an `x_s2d` the caller has already filled (scene tiles, letterboxed images) -> the shared
        output, plan-owned as in forward().  Plain plans only: the augmented branches resample the image itself."""
        if self.augment:
            raise RuntimeError("forward_s2d runs the plain ensemble plan; test-time augmentation resamples the image in forward()")
        with torch.cuda.device(self.device):
            for _, fn in self.steps[1:]:
                fn(None)
        return self.pred
