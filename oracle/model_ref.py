"""fp32 PyTorch restatement of the reference forward pass — TEST INFRASTRUCTURE (torch fp32 reference
for a floating-point kernel; never imported by the product package).

Follows models/common.py:37-49 (Conv), :94-104 (Bottleneck), :126-138 (C3), :181-196
(SPPF), :267-274 (Concat), nn.Upsample, models/yolo.py:49-81 (Detect) and :163-181
(_forward_once), operating on the parameter containers of yolov5_obb_b200.yolo.Model (same names and
shapes as the reference modules).  Pinned by tests/golden/model_golden.npz, which holds outputs of the
REFERENCE model itself for the same seed (tests/golden/make_model_golden.py).
"""
import torch
import torch.nn.functional as F

from yolov5_obb_b200 import yolo as Y


class _RoundBf16(torch.autograd.Function):
    """Value AND gradient rounded to bf16: the storage rounding points of the device path, used to measure the
    noise floor bf16 storage puts under a comparison with this fp32 oracle (never a parity target itself)."""

    @staticmethod
    def forward(ctx, t):
        return t.bfloat16().float()

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


_EMULATE_BF16 = False


def _r(t):
    return _RoundBf16.apply(t) if _EMULATE_BF16 else t


def conv_fwd(m: Y.Conv, x, training=False):
    y = _r(F.conv2d(x, _r(m.conv.weight), m.conv.bias, m.conv.stride, m.conv.padding))
    if hasattr(m, "bn") and m.bn is not None:
        bn = m.bn
        y = F.batch_norm(y, bn.running_mean, bn.running_var, bn.weight, bn.bias, training, bn.momentum, bn.eps)
    return _r(F.silu(y) if isinstance(m.act, torch.nn.SiLU) else y)


def bottleneck_fwd(m: Y.Bottleneck, x, training=False):
    y = conv_fwd(m.cv2, conv_fwd(m.cv1, x, training), training)
    return _r(x + y) if m.add else y


def c3_fwd(m: Y.C3, x, training=False):
    y = conv_fwd(m.cv1, x, training)
    for b in m.m:
        y = bottleneck_fwd(b, y, training)
    return conv_fwd(m.cv3, torch.cat((y, conv_fwd(m.cv2, x, training)), 1), training)


def sppf_fwd(m: Y.SPPF, x, training=False):
    x = conv_fwd(m.cv1, x, training)
    y1 = F.max_pool2d(x, 5, 1, 2)
    y2 = F.max_pool2d(y1, 5, 1, 2)
    return conv_fwd(m.cv2, torch.cat([x, y1, y2, F.max_pool2d(y2, 5, 1, 2)], 1), training)


def detect_fwd(m: Y.Detect, xs, training=False):
    z, outs = [], []
    for i in range(m.nl):
        x = F.conv2d(xs[i], _r(m.m[i].weight), m.m[i].bias)
        bs, _, ny, nx = x.shape
        x = x.view(bs, m.na, m.no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()
        outs.append(x)
        if not training:
            yv, xv = torch.meshgrid(torch.arange(ny, device=x.device), torch.arange(nx, device=x.device), indexing="ij")
            grid = torch.stack((xv, yv), 2).expand((1, m.na, ny, nx, 2)).float()
            anchor_grid = (m.anchors[i].clone() * m.stride[i]).view((1, m.na, 1, 1, 2)).expand((1, m.na, ny, nx, 2)).float()
            y = x.sigmoid()
            y[..., 0:2] = (y[..., 0:2] * 2 - 0.5 + grid) * m.stride[i]
            y[..., 2:4] = (y[..., 2:4] * 2) ** 2 * anchor_grid
            z.append(y.view(bs, -1, m.no))
    return outs if training else (torch.cat(z, 1), outs)


def forward_with_grad(model: Y.Model, x: torch.Tensor, training: bool = False, return_layers: bool = False,
                      emulate_bf16: bool = False):
    """models/yolo.py:163-181 over the container modules.  x: [B,3,H,W] fp32.  Differentiable (autograd is the
    oracle of the backward pass, as it is the reference's own backward under train.py:333).
    emulate_bf16=True rounds weights, conv outputs, activations (and their gradients) to bf16 where the device path
    stores bf16: tests use the distance between the two oracle variants as the noise floor of the comparison."""
    global _EMULATE_BF16
    _EMULATE_BF16 = bool(emulate_bf16)
    try:
        return _forward_impl(model, _r(x), training, return_layers)
    finally:
        _EMULATE_BF16 = False


def _forward_impl(model, x, training, return_layers):
    ys = []
    for m in model.model:
        if m.f != -1:
            x = ys[m.f] if isinstance(m.f, int) else [x if j == -1 else ys[j] for j in m.f]
        if isinstance(m, Y.Conv):
            x = conv_fwd(m, x, training)
        elif isinstance(m, Y.C3):
            x = c3_fwd(m, x, training)
        elif isinstance(m, Y.SPPF):
            x = sppf_fwd(m, x, training)
        elif isinstance(m, Y.Concat):
            x = torch.cat(x, m.d)
        elif isinstance(m, Y.Upsample):
            x = F.interpolate(x, scale_factor=2, mode="nearest")
        elif isinstance(m, Y.Detect):
            x = detect_fwd(m, x, training)
        ys.append(x)
    return (x, ys) if return_layers else x


@torch.no_grad()
def forward(model: Y.Model, x: torch.Tensor, training: bool = False, return_layers: bool = False,
            emulate_bf16: bool = False):
    return forward_with_grad(model, x, training, return_layers, emulate_bf16)
