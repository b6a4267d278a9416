"""CPU restatement of the image front end of detect.py / val.py, in numpy only (no cv2, no torch):

* resize(): cv2.resize for uint8 HWC images with INTER_LINEAR (the 8-bit fixed-point path: 11-bit coefficients, int32
  horizontal pass, the `>> 4`, `>> 16`, `+ 2 >> 2` vertical pass), its silent switch to INTER_AREA when both scale factors
  are exactly 2, and INTER_AREA for shrinking: the integer-factor path (2x2 rounds half up in integers, every other block
  rounds the fp32 product sum * (1.f / area) half to even) and the fractional path (fp32 weights accumulated per
  destination pixel in OpenCV's order: columns first, rows second, each product and sum rounded separately);
* letterbox() (utils/augmentations.py:92-128), LoadImages' transpose (utils/datasets.py:224-228), load_image_label's resize
  (utils/datasets.py:714-718) and the rect batch shapes (utils/datasets.py:472-492).

tests/test_letterbox_cpu.py pins this against the installed cv2 over a sweep of size pairs and against the reference's own
functions (tests/golden/letterbox_golden.npz); the GPU tests compare the kernels against it."""
import math

import numpy as np

LINEAR, AREA = "linear", "area"
COEF_BITS = 11
COEF_ONE = 1 << COEF_BITS
DBL_EPSILON = 2.220446049250313e-16


def _scale(src: int, dst: int) -> float:
    return 1.0 / (dst / float(src))   # inv_scale = dsize / ssize in double, scale = 1. / inv_scale


def _cv_round(x: float) -> int:
    return int(np.rint(x))


def _is_int_scale(scale: float) -> bool:
    return abs(scale - _cv_round(scale)) < DBL_EPSILON


def linear_tab(src: int, dst: int, clamp_frac: bool):
    """(first source index, coefficient pairs int16 [dst, 2]) of one axis.  Columns (clamp_frac) move an index outside the
    image to the border pixel with fraction 0; rows keep their fraction and clip the two row indices instead."""
    scale = _scale(src, dst)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp_frac:
        lo, hi = s < 0, s >= src - 1
        f[lo | hi] = 0
        s[lo] = 0
        s[hi] = src - 1
    one = np.float32(1.0)
    k = np.float32(COEF_ONE)
    coef = np.stack([np.rint((one - f) * k), np.rint(f * k)], 1).astype(np.int32)
    return s, coef


def resize_linear(img: np.ndarray, new_w: int, new_h: int) -> np.ndarray:
    h0, w0 = img.shape[:2]
    sx, a = linear_tab(w0, new_w, True)
    sy, b = linear_tab(h0, new_h, False)
    sx1 = np.minimum(sx + 1, w0 - 1)
    S = img.astype(np.int32)
    hp = S[:, sx] * a[None, :, 0, None] + S[:, sx1] * a[None, :, 1, None]        # [h0, new_w, 3] int32
    r0, r1 = np.clip(sy, 0, h0 - 1), np.clip(sy + 1, 0, h0 - 1)
    v = ((b[:, 0, None, None] * (hp[r0] >> 4)) >> 16) + ((b[:, 1, None, None] * (hp[r1] >> 4)) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def area_tab(src: int, dst: int):
    """computeResizeAreaTab: per destination index the list of (source index, fp32 weight)."""
    scale = _scale(src, dst)
    out = []
    for d in range(dst):
        f1 = d * scale
        f2 = f1 + scale
        cell = min(scale, src - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, src - 1)
        s1 = min(s1, s2)
        e = []
        if s1 - f1 > 1e-3:
            e.append((s1 - 1, np.float32((s1 - f1) / cell)))
        for s in range(s1, s2):
            e.append((s, np.float32(1.0 / cell)))
        if f2 - s2 > 1e-3:
            e.append((s2, np.float32(min(min(f2 - s2, 1.0), cell) / cell)))
        out.append(e)
    return out


def _dense(tab):
    k = max(len(e) for e in tab)
    si = np.zeros((len(tab), k), np.int64)
    al = np.zeros((len(tab), k), np.float32)
    n = np.zeros(len(tab), np.int64)
    for d, e in enumerate(tab):
        n[d] = len(e)
        for j, (s, a) in enumerate(e):
            si[d, j], al[d, j] = s, a
    return si, al, n


def resize_area(img: np.ndarray, new_w: int, new_h: int) -> np.ndarray:
    h0, w0 = img.shape[:2]
    if new_w > w0 or new_h > h0:
        raise ValueError("INTER_AREA is restated for shrinking only")
    sx, sy = _scale(w0, new_w), _scale(h0, new_h)
    if _is_int_scale(sx) and _is_int_scale(sy):
        kx, ky = _cv_round(sx), _cv_round(sy)
        blocks = img[:new_h * ky, :new_w * kx].astype(np.int32).reshape(new_h, ky, new_w, kx, 3).sum((1, 3))
        if kx == 2 and ky == 2:
            return ((blocks + 2) >> 2).astype(np.uint8)
        scale = np.float32(1.0) / np.float32(kx * ky)
        return np.clip(np.rint(blocks.astype(np.float32) * scale), 0, 255).astype(np.uint8)
    xi, xa, xn = _dense(area_tab(w0, new_w))
    yi, ya, yn = _dense(area_tab(h0, new_h))
    S = img.astype(np.float32)
    buf = np.zeros((h0, new_w, 3), np.float32)
    for j in range(xi.shape[1]):                       # columns, in table order; padded taps add 0 * S = +0
        buf = buf + S[:, xi[:, j]] * xa[None, :, j, None]
    acc = ya[:, 0, None, None] * buf[yi[:, 0]]
    for j in range(1, yi.shape[1]):
        t = acc + ya[:, j, None, None] * buf[yi[:, j]]
        acc = np.where((j < yn)[:, None, None], t, acc)
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def resize(img: np.ndarray, size_wh, interp: str) -> np.ndarray:
    """cv2.resize(img, (w, h), interpolation=INTER_LINEAR | INTER_AREA) for uint8 [H, W, 3]."""
    new_w, new_h = int(size_wh[0]), int(size_wh[1])
    h0, w0 = img.shape[:2]
    if interp == LINEAR:
        sx, sy = _scale(w0, new_w), _scale(h0, new_h)
        if _is_int_scale(sx) and _is_int_scale(sy) and _cv_round(sx) == 2 and _cv_round(sy) == 2:
            return resize_area(img, new_w, new_h)
        return resize_linear(img, new_w, new_h)
    if interp == AREA:
        return resize_area(img, new_w, new_h)
    raise ValueError(interp)


# ------------------------------------------------------------------------------------------------ geometry
def letterbox_geometry(shape0, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """utils/augmentations.py:100-126 -> new_unpad (w, h), (top, bottom, left, right), ratio (w, h), (dw, dh)."""
    shape = (int(shape0[0]), int(shape0[1]))
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scaleFill:
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    return new_unpad, (top, bottom, left, right), ratio, (dw, dh)


def letterbox(im, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    new_unpad, (top, bottom, left, right), ratio, pad = letterbox_geometry(im.shape[:2], new_shape, auto, scaleFill, scaleup,
                                                                          stride)
    if im.shape[:2][::-1] != new_unpad:
        im = resize(im, new_unpad, LINEAR)
    h, w = im.shape[:2]
    out = np.empty((h + top + bottom, w + left + right, 3), np.uint8)
    out[:] = np.asarray(color, np.uint8)
    out[top:top + h, left:left + w] = im
    return out, ratio, pad


def to_chw_rgb(im: np.ndarray) -> np.ndarray:
    """utils/datasets.py:227-228: HWC BGR -> CHW RGB, contiguous."""
    return np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])


def load_image_size(h0: int, w0: int, img_size: int, augment: bool = False):
    """utils/datasets.py:714-718 -> ((h, w) after the resize, interpolation or None when r == 1, r)."""
    r = img_size / max(h0, w0)
    if r == 1:
        return (h0, w0), None, r
    return (int(h0 * r), int(w0 * r)), (AREA if r < 1 and not augment else LINEAR), r


def load_image(im: np.ndarray, img_size: int, augment: bool = False):
    h0, w0 = im.shape[:2]
    (h, w), interp, _ = load_image_size(h0, w0, img_size, augment)
    if interp is not None:
        im = resize(im, (w, h), interp)
    return im, (h0, w0), im.shape[:2]


def rect_batch_shapes(shapes_wh, batch_size: int, img_size: int, stride: int = 32, pad: float = 0.0):
    """utils/datasets.py:450,472-492: shapes_wh [n, 2] (w, h) -> (order, batch index per sorted image, batch_shapes [nb, 2]
    (h, w))."""
    s = np.array(shapes_wh, dtype=np.float64)
    n = len(s)
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    ar = s[:, 1] / s[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    return irect, bi, np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride


def rect_item(im: np.ndarray, img_size: int, batch_shape):
    """LoadImagesAndLabels.__getitem__ without augmentation (utils/datasets.py:585-590, 662-663): -> (CHW RGB image,
    shapes entry ((h0, w0), ((h / h0, w / w0), pad)), r of the first resize, ratio of the letterbox)."""
    img, (h0, w0), (h, w) = load_image(im, img_size)
    r = img_size / max(h0, w0)
    img, ratio, pad = letterbox(img, tuple(int(v) for v in batch_shape), auto=False, scaleup=False)
    return to_chw_rgb(img), ((h0, w0), ((h / h0, w / w0), pad)), r, ratio
