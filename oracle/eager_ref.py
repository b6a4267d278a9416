"""Eager PyTorch (cuDNN) restatement of the reference's GPU inference path — TEST / BENCH INFRASTRUCTURE, never imported by
the product package.  This is "the bar to beat" of SURVEY §2.3 L1: what `val.py --task speed` runs on a GPU:

  * the fused model (attempt_load(..., fuse=True) -> Conv.forward_fuse, models/common.py:48-49: act(conv(x)) with BatchNorm
    folded into the conv, utils/torch_utils.py:192-212), in fp16 (`model.half()`, val.py:128,142) with cudnn.benchmark=True,
    NCHW (the reference never sets channels_last);
  * Detect exactly as models/yolo.py:49-81 (oracle.model_ref.detect_fwd);
  * non_max_suppression_obb (utils/general.py:772-862) as the per-image Python loop over the reference's own CUDA kernel K1
    (utils/nms_rotated/src/nms_rotated_cuda.cu compiled by oracle/build_ref.py into oracle/_ref).
"""
import torch
import torch.nn.functional as F

from yolov5_obb_b200 import yolo as Y
from . import model_ref


class EagerFusedModel:
    def __init__(self, model: Y.Model, device, half: bool = True):
        self.model = model
        self.dtype = torch.float16 if half else torch.float32
        self.device = torch.device(device)
        self.w = {}
        for m in model.modules():
            if isinstance(m, Y.Conv):
                bn = m.bn
                scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
                w = m.conv.weight.detach().float() * scale.view(-1, 1, 1, 1)
                b = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
                self.w[id(m)] = (w.to(self.device, self.dtype), b.to(self.device, self.dtype))
        det = model.model[-1]
        self.det_w = [(mi.weight.detach().to(self.device, self.dtype), mi.bias.detach().to(self.device, self.dtype)) for mi in det.m]
        self.anchors = det.anchors.detach().to(self.device)
        self.stride = det.stride.detach().to(self.device)

    def _conv(self, m, x):
        w, b = self.w[id(m)]
        y = F.conv2d(x, w, b, m.conv.stride, m.conv.padding)
        return F.silu(y) if isinstance(m.act, torch.nn.SiLU) else y

    def _c3(self, m, x):
        y = self._conv(m.cv1, x)
        for b in m.m:
            z = self._conv(b.cv2, self._conv(b.cv1, y))
            y = y + z if b.add else z
        return self._conv(m.cv3, torch.cat((y, self._conv(m.cv2, x)), 1))

    def _sppf(self, m, x):
        x = self._conv(m.cv1, x)
        y1 = F.max_pool2d(x, 5, 1, 2)
        y2 = F.max_pool2d(y1, 5, 1, 2)
        return self._conv(m.cv2, torch.cat([x, y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1))

    def _detect(self, det, xs):
        z = []
        for i in range(det.nl):
            w, b = self.det_w[i]
            x = F.conv2d(xs[i], w, b)
            bs, _, ny, nx = x.shape
            x = x.view(bs, det.na, det.no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
            yv, xv = torch.meshgrid(torch.arange(ny, device=x.device), torch.arange(nx, device=x.device), indexing="ij")
            grid = torch.stack((xv, yv), 2).expand((1, det.na, ny, nx, 2)).float()
            ag = (self.anchors[i].clone() * self.stride[i]).view((1, det.na, 1, 1, 2)).expand((1, det.na, ny, nx, 2)).float()
            y = x.sigmoid()
            y[..., 0:2] = (y[..., 0:2] * 2 - 0.5 + grid) * self.stride[i]
            y[..., 2:4] = (y[..., 2:4] * 2) ** 2 * ag
            z.append(y.view(bs, -1, det.no))
        return torch.cat(z, 1)

    @torch.no_grad()
    def forward(self, x):
        """x: [B,3,H,W] in [0,1], self.dtype, on self.device -> pred [B, A, no] (models/yolo.py:163-181)."""
        ys = []
        for m in self.model.model:
            if m.f != -1:
                x = ys[m.f] if isinstance(m.f, int) else [x if j == -1 else ys[j] for j in m.f]
            if isinstance(m, Y.Conv):
                x = self._conv(m, x)
            elif isinstance(m, Y.C3):
                x = self._c3(m, x)
            elif isinstance(m, Y.SPPF):
                x = self._sppf(m, x)
            elif isinstance(m, Y.Concat):
                x = torch.cat(x, m.d)
            elif isinstance(m, Y.Upsample):
                x = F.interpolate(x, scale_factor=2, mode="nearest")
            elif isinstance(m, Y.Detect):
                x = self._detect(m, x)
            ys.append(x if m.i in self.model.save else None)  # models/yolo.py:179
        return x
