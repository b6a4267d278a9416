"""fp32 PyTorch restatement of the reference's test-time augmentation — TEST INFRASTRUCTURE (never imported by the product
package).

models/yolo.py:149-161 (_forward_augment), :183-198 (_descale_pred, the `inplace` branch), :200-209 (_clip_augmented) and
utils/torch_utils.py:239-249 (scale_img), on top of oracle/model_ref.forward.  The de-scale uses the reference's own torch ops,
so on the CPU `p[..., :4] /= s` divides.  Pinned by tests/golden/tta_golden.npz, which holds the REFERENCE model's own
`Model(...)(x, augment=True)` for the same seed (tests/golden/make_tta_golden.py).
"""
import math

import torch
import torch.nn.functional as F

from oracle import model_ref

SCALES = (1, 0.83, 0.67)
FLIPS = (None, 3, None)


def scale_img(img, ratio=1.0, same_shape=False, gs=32):
    if ratio == 1.0:
        return img
    h, w = img.shape[2:]
    s = (int(h * ratio), int(w * ratio))
    img = F.interpolate(img, size=s, mode="bilinear", align_corners=False)
    if not same_shape:
        h, w = (math.ceil(x * ratio / gs) * gs for x in (h, w))
    return F.pad(img, [0, w - s[1], 0, h - s[0]], value=0.447)


def descale_pred(p, flips, scale, img_size):
    p[..., :4] /= scale
    if flips == 2:
        p[..., 1] = img_size[0] - p[..., 1]
    elif flips == 3:
        p[..., 0] = img_size[1] - p[..., 0]
    return p


def clip_augmented(y, nl=3):
    g = sum(4 ** x for x in range(nl))
    e = 1
    i = (y[0].shape[1] // g) * sum(4 ** x for x in range(e))
    y[0] = y[0][:, :-i]
    i = (y[-1].shape[1] // g) * sum(4 ** (nl - 1 - x) for x in range(e))
    y[-1] = y[-1][:, i:]
    return y


@torch.no_grad()
def forward_augment(model, x: torch.Tensor, emulate_bf16: bool = False):
    """x [B, 3, H, W] fp32 -> (pred [B, A_tta, no], None), as Model._forward_augment returns it."""
    img_size = x.shape[-2:]
    y = []
    for si, fi in zip(SCALES, FLIPS):
        xi = scale_img(x.flip(fi) if fi else x, si, gs=int(model.stride.max()))
        yi = model_ref.forward(model, xi, emulate_bf16=emulate_bf16)[0]
        y.append(descale_pred(yi, fi, si, img_size))
    y = clip_augmented(y, model.model[-1].nl)
    return torch.cat(y, 1), None
