"""Host-side mirror of utils/loss.py:90-192 ComputeLoss — same constructor and call
signature, autograd-compatible (`scaler.scale(loss).backward()`, train.py:333), backed by csrc/loss.cu.

    compute_loss = ComputeLoss(model)            # reads model.hyp and the Detect module
    loss, loss_items = compute_loss(pred, targets)   # pred: list of [B,3,H,W,no]; targets [nt,187]

Focal loss (fl_gamma > 0) is outside the hot path (every shipped hyp sets 0,
data/hyps/obb/hyp.finetune_dota.yaml:19) and is refused loudly.
"""
import ctypes
from ctypes import c_void_p, c_int, c_int64, c_float

import torch

from . import _lib
from .general import require_nc

MAX_LEVELS = 4  # Y5OBB_LOSS_MAX_LEVELS (include/y5obb.h): the P3-P6 Detect of models/hub/yolov5*6.yaml


class LossDesc(ctypes.Structure):
    """Mirror of y5obb_loss_desc (include/y5obb.h)."""
    _fields_ = [
        ("p", c_void_p * MAX_LEVELS), ("grad", c_void_p * MAX_LEVELS), ("H", c_int * MAX_LEVELS), ("W", c_int * MAX_LEVELS),
        ("stride", c_float * MAX_LEVELS), ("anchors", c_float * (MAX_LEVELS * 3 * 2)), ("balance", c_float * MAX_LEVELS),
        ("nl", c_int), ("B", c_int), ("na", c_int), ("no", c_int), ("nc", c_int),
        ("targets", c_void_p), ("nt", c_int), ("tcols", c_int),
        ("anchor_t", c_float), ("cp", c_float), ("cn", c_float),
        ("hyp_box", c_float), ("hyp_obj", c_float), ("hyp_cls", c_float), ("hyp_theta", c_float),
        ("cls_pw", c_float), ("obj_pw", c_float), ("theta_pw", c_float), ("csl_sigma", c_float),
    ]


class LossHead(ctypes.Structure):
    """Mirror of y5obb_loss_head (include/y5obb.h)."""
    _fields_ = [
        ("feat", c_void_p * MAX_LEVELS), ("pix_stride", c_int64 * MAX_LEVELS), ("row_stride", c_int64 * MAX_LEVELS),
        ("img_stride", c_int64 * MAX_LEVELS), ("H", c_int * MAX_LEVELS), ("W", c_int * MAX_LEVELS), ("C", c_int * MAX_LEVELS),
        ("w", c_void_p * MAX_LEVELS), ("bias", c_void_p * MAX_LEVELS),
    ]


def smooth_BCE(eps=0.1):  # utils/loss.py:13-15
    return 1.0 - 0.5 * eps, 0.5 * eps


class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, owner, targets, *p):
        L = _lib.lib()
        dev = p[0].device
        ps = [x.contiguous() for x in p]
        tg = targets.detach().float().contiguous()
        d = owner._desc(ps, tg)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        items = torch.empty(4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            nbytes = L.y5obb_loss_workspace_bytes(ctypes.byref(d))
            if nbytes == 0:
                raise RuntimeError("y5obb_loss_workspace_bytes: invalid loss description")
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)  # kept for backward (holds the matched rows)
            rc = L.y5obb_loss_forward(ctypes.byref(d), loss.data_ptr(), items.data_ptr(), ws.data_ptr(), ws.numel(),
                                      _lib.stream_ptr(dev))
        _lib.check(rc, "y5obb_loss_forward")
        ctx.owner, ctx.ws, ctx.tg = owner, ws, tg
        ctx.save_for_backward(*ps)
        ctx.mark_non_differentiable(items)
        return loss, items

    @staticmethod
    def backward(ctx, g_loss, _g_items):
        L = _lib.lib()
        ps = ctx.saved_tensors
        dev = ps[0].device
        grads = [torch.empty_like(x) for x in ps]
        d = ctx.owner._desc(list(ps), ctx.tg, grads)
        g = g_loss.detach().float().contiguous()
        with torch.cuda.device(dev):
            rc = L.y5obb_loss_backward(ctypes.byref(d), g.data_ptr(), ctx.ws.data_ptr(), ctx.ws.numel(),
                                       _lib.stream_ptr(dev))
        _lib.check(rc, "y5obb_loss_backward")
        return (None, None, *grads)


class ComputeLoss:
    # Compute losses (utils/loss.py:90)
    def __init__(self, model, autobalance=False):
        self.sort_obj_iou = False
        h = model.hyp  # hyperparameters
        if h.get("fl_gamma", 0.0) > 0:
            raise RuntimeError("FocalLoss (fl_gamma > 0) is not part of the hot path")
        if autobalance:
            raise RuntimeError("autobalance reads the loss on the host every step; not part of the hot path")
        self.cp, self.cn = smooth_BCE(eps=h.get("label_smoothing", 0.0))
        m = model.module if hasattr(model, "module") else model
        det = m.model[-1]  # Detect() module
        self.stride = det.stride
        self.balance = {3: [4.0, 1.0, 0.4]}.get(det.nl, [4.0, 1.0, 0.25, 0.06, 0.02])
        self.gr, self.hyp, self.autobalance = 1.0, h, autobalance
        for k in "na", "nc", "nl", "anchors":
            setattr(self, k, getattr(det, k))
        require_nc(self.nc, "ComputeLoss")
        if self.nl not in (3, MAX_LEVELS) or self.na > 3:
            raise RuntimeError(f"the loss takes the 3-level Detect of yolov5{{n,s,m,l,x}}.yaml or the {MAX_LEVELS}-level one of "
                               f"models/hub/yolov5{{n,s,m,l,x}}6.yaml, with at most 3 anchors per level; this one has "
                               f"nl={self.nl}, na={self.na}")
        self._anchors_host = [float(v) for v in self.anchors.detach().float().cpu().flatten().tolist()]
        self._stride_host = [float(s) for s in self.stride]

    def _desc(self, ps, tg, grads=None) -> LossDesc:
        no = ps[0].shape[-1]
        d = self._base_desc(ps[0].shape[0], no, tg)
        for i, x in enumerate(ps):
            if x.dtype != torch.float32 or x.dim() != 5 or x.shape[-1] != no:
                raise RuntimeError("predictions must be fp32 [B, na, H, W, no] tensors")
            d.p[i] = x.data_ptr()
            d.H[i], d.W[i] = x.shape[2], x.shape[3]
            if grads is not None:
                d.grad[i] = grads[i].data_ptr()
        return d

    def _base_desc(self, B, no, tg) -> LossDesc:
        """Everything but the logits and their shapes."""
        d = LossDesc()
        for i in range(self.nl):
            d.stride[i] = self._stride_host[i]
            d.balance[i] = self.balance[i]
        for i, v in enumerate(self._anchors_host):
            d.anchors[i] = v
        d.nl, d.B, d.na, d.no, d.nc = self.nl, B, self.na, no, self.nc
        d.targets, d.nt, d.tcols = (tg.data_ptr() if tg.numel() else None), tg.shape[0], tg.shape[1] if tg.dim() == 2 else 187
        h = self.hyp
        d.anchor_t, d.cp, d.cn = h["anchor_t"], self.cp, self.cn
        d.hyp_box, d.hyp_obj, d.hyp_cls, d.hyp_theta = h["box"], h["obj"], h["cls"], h["theta"]
        d.cls_pw, d.obj_pw, d.theta_pw = h.get("cls_pw", 1.0), h.get("obj_pw", 1.0), h.get("theta_pw", 1.0)
        d.csl_sigma = float(h.get("csl_radius", 2.0))
        if d.tcols not in (7, 8) and d.tcols < 187:
            raise RuntimeError("targets must have 187 columns (reference layout), or 8 (.., theta, csl index) or 7 (.., theta)")
        return d

    def __call__(self, p, targets):  # predictions, targets
        """
        Args:
            p (list[P3_out,...]): torch.Size(b, self.na, h_i, w_i, self.no)
            targets (tensor): (n_gt_all_batch, [img_index clsid cx cy l s theta gaussian_θ_labels])
                compact forms (8f rank 2): [nt, 8] = (..., theta, csl_index) with csl_index = compact_csl_index(theta) below, or
                [nt, 7] = (..., theta): the Circular-Smooth-Label row is rebuilt inside the kernel
        Return:
            total_loss * bs (tensor): [1];  torch.cat((lbox, lobj, lcls, ltheta)).detach(): [4]
        """
        for x in p:
            _lib.require_cuda(x, "prediction")
        _lib.require_cuda(targets, "targets")
        ps = [x.float() for x in p]  # AMP half predictions are widened; autograd casts the gradient back
        return _LossFn.apply(self, targets, *ps)


    def head_items(self, engine, targets):
        """val.py:198-199's `compute_loss([x.float() for x in train_out], targets)[1]` for the eval forward an
        engine.InferenceEngine (Model.records_plan) has just run, without its raw head output: the loss reads logits computed
        from the Detect inputs the plan keeps (y5obb_loss_forward_head; for an fp16 plan y5obb_loss_forward_head_f16, whose
        logits are rounded to fp16 as the half Detect conv's are).  targets: CUDA [nt, 187 | 8 | 7] as in __call__.
        Returns device (loss [1], items [4]) = (lbox, lobj, lcls, ltheta); asynchronous, no autograd.  The features must still
        be those of the batch the targets belong to: call it before the plan's next forward."""
        from .engine import InferenceEngine
        if not isinstance(engine, InferenceEngine):
            raise RuntimeError(f"head_items needs an engine.InferenceEngine (one scale, every Detect level), got "
                               f"{type(engine).__name__}")
        if engine.levels != tuple(range(self.nl)):
            raise RuntimeError(f"the plan emits Detect levels {engine.levels}; the loss needs all {self.nl}")
        if (engine.det_nl, engine.na, engine.nc, engine.det_anchors, engine.det_strides) != (
                self.nl, self.na, self.nc, self._anchors_host, self._stride_host):
            raise RuntimeError("the plan's Detect (nl, na, nc, anchors, strides) differs from the one this loss was built for")
        _lib.require_cuda(targets, "targets")
        dev = engine.device
        if targets.device != dev:
            raise RuntimeError(f"targets are on {targets.device}, the plan on {dev}")
        tg = targets.detach().float().contiguous()
        d = self._base_desc(engine.B, engine.no, tg)
        h = LossHead()
        for i, (x, w, b) in enumerate(engine.head_inputs()):
            h.feat[i] = x.ptr
            h.pix_stride[i], h.row_stride[i], h.img_stride[i] = x.pix_stride, x.W * x.pix_stride, x.H * x.W * x.pix_stride
            h.H[i], h.W[i], h.C[i] = x.H, x.W, x.C
            h.w[i], h.bias[i] = w.data_ptr(), b.data_ptr()
        L = _lib.lib()
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        items = torch.empty(4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            nbytes = L.y5obb_loss_head_workspace_bytes(ctypes.byref(d), ctypes.byref(h))
            if nbytes == 0:
                raise RuntimeError("y5obb_loss_head_workspace_bytes: invalid loss description or Detect inputs")
            st = _lib.stream_ptr(dev)
            ws = _lib.workspace(nbytes, dev, f"loss_head:{st}")
            name = "y5obb_loss_forward_head_f16" if engine.half else "y5obb_loss_forward_head"
            _lib.check(getattr(L, name)(ctypes.byref(d), ctypes.byref(h), loss.data_ptr(), items.data_ptr(),
                                        ws.data_ptr(), ws.numel(), st), name)
        return loss, items


def compact_csl_index(theta_rad, num_class: int = 180):
    """Column 7 of the 8-column compact target layout: the rotation index of utils/rboxs_utils.py:21,
    `int(num_class / 2 - angle)` with `angle = theta * 180 / 3.141592 + 90` (:70, :5), evaluated in fp64 on the host exactly as
    the reference's dataloader does.  theta_rad: float64 numpy array (the values poly2rbox returned)."""
    import numpy as np
    angle = np.asarray(theta_rad, dtype=np.float64) * 180 / 3.141592 + 90
    return np.trunc(num_class / 2 - angle).astype(np.float32)
