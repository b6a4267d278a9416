"""Images of any size on the device: the host geometry of detect.py's and val.py's loaders, the packing of a batch of
source images for csrc/letterbox.cu, and the batched rbox2poly + scale_polys that brings detections back to source pixels.

The reference does all of it on the CPU, per image: cv2.resize + copyMakeBorder + transpose (utils/augmentations.py:92-128,
utils/datasets.py:217-229 and :585-590,662-663,702-720) before the forward and rbox2poly + scale_polys after NMS
(detect.py:129-147, val.py:226-232).  Here only the O(width + height) geometry stays on the host: letterbox_geometry,
load_image_size and rect_batch_shapes return the reference's values, pack_batch ships the decoded images as they are with one
descriptor and two coefficient tables each, and y5obb_letterbox_s2d_u8 writes the stem input of the whole batch
(letterboxed_records runs it and the records plan for DetectPipeline.run_images and the Validator's raw form).  The tables
are formed in the float types OpenCV uses (DESIGN.md section 4), so the resampled bytes are OpenCV's."""
import functools
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .general import DetectRecords

LINEAR, AREA = "linear", "area"
MODE_COPY, MODE_LINEAR, MODE_AREA_INT, MODE_AREA = 0, 1, 2, 3   # Y5OBB_LB_*
DESC_WORDS = 16                                                 # sizeof(y5obb_letterbox_desc) / 4
_DBL_EPSILON = 2.220446049250313e-16


# ---------------------------------------------------------------------------------------------------------------- geometry
def letterbox_geometry(shape0, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """utils/augmentations.py:100-126 for an image of shape0 = (h, w): -> new_unpad (w, h), (top, bottom, left, right),
    ratio (w, h), (dw, dh), value for value (round(d - 0.1) / round(d + 0.1), np.mod under auto, scaleFill)."""
    shape = (int(shape0[0]), int(shape0[1]))
    if shape[0] < 1 or shape[1] < 1:
        raise RuntimeError(f"empty image {shape}")
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


def load_image_size(h0: int, w0: int, img_size: int, augment: bool = False):
    """load_image_label's resize (utils/datasets.py:714-718): -> ((h, w), interpolation or None when r == 1, r)."""
    r = img_size / max(h0, w0)
    if r == 1:
        return (h0, w0), None, r
    return (int(h0 * r), int(w0 * r)), (AREA if r < 1 and not augment else LINEAR), r


def rect_batch_shapes(shapes_wh, batch_size: int, img_size: int, stride: int = 32, pad: float = 0.0):
    """The rect batching of LoadImagesAndLabels (utils/datasets.py:450,472-492): shapes_wh [n, 2] (w, h) of the source images ->
    (order, batch_shapes): `order` the aspect-ratio sort (np.argsort, as the reference), image order[k] goes to batch
    k // batch_size; batch_shapes [nb, 2] int (h, w) = ceil(shape ratios * img_size / stride + pad) * stride."""
    s = np.array(shapes_wh, dtype=np.float64).reshape(-1, 2)
    n = len(s)
    if n == 0:
        raise RuntimeError("no images")
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    ar = s[:, 1] / s[:, 0]
    order = ar.argsort()
    ar = ar[order]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    return order, np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride


class Placement:
    """Where one source image lands in the letterboxed batch image: resampled size, interpolation, border offsets, and what
    the reference keeps for the way back: `ratio` (w, h) and `pad` (dw, dh) of letterbox, `r` of load_image_label's resize
    and `shapes` = ((h0, w0), ((h / h0, w / w0), pad)) (utils/datasets.py:590).  `pad_gain` = (pad_x, pad_y, gain) is what
    scale_polys divides the detections by: from `shapes` as val.py:232 passes it, unless the caller sets detect.py's."""

    def __init__(self, h0, w0, new_h, new_w, top, left, interp, ratio, pad, r=1.0, hw=None):
        self.h0, self.w0, self.new_h, self.new_w, self.top, self.left = h0, w0, new_h, new_w, top, left
        self.interp, self.ratio, self.pad, self.r = interp, ratio, pad, r
        h, w = hw if hw is not None else (h0, w0)
        self.shapes = ((h0, w0), ((h / h0, w / w0), pad))
        self.pad_gain = (pad[0], pad[1], self.shapes[1][0][0])   # scale_polys: gain = ratio_pad[0][0], pad = ratio_pad[1]

    def map_labels(self, polys: np.ndarray) -> np.ndarray:
        """Label polygons [n, 8] (x1 y1 ... x4 y4) in source pixels -> network-input pixels, as utils/datasets.py:719 and
        :595-596 move them: `* r`, then `* ratio + pad`."""
        out = np.array(polys, dtype=np.float64, copy=True).reshape(-1, 8)
        out *= self.r
        out[:, 0::2] = out[:, 0::2] * self.ratio[0] + self.pad[0]
        out[:, 1::2] = out[:, 1::2] * self.ratio[1] + self.pad[1]
        return out


def place_detect(h0: int, w0: int, img_size=1024, stride: int = 32, auto: bool = True, scaleFill: bool = False,
                 scaleup: bool = True) -> Tuple[Placement, Tuple[int, int]]:
    """LoadImages (detect.py): letterbox(img0, img_size, stride=stride, auto=auto) -> (Placement, (Hp, Wp))."""
    (nw, nh), (top, bottom, left, right), ratio, pad = letterbox_geometry((h0, w0), img_size, auto, scaleFill, scaleup, stride)
    if nw < 1 or nh < 1:
        raise RuntimeError(f"a {h0} x {w0} image letterboxed to {img_size} has no pixels left ({nh} x {nw})")
    p, hw = Placement(h0, w0, nh, nw, top, left, LINEAR, ratio, pad), (nh + top + bottom, nw + left + right)
    p.pad_gain = detect_pad_gain(hw, (h0, w0))
    return p, hw


def place_rect(h0: int, w0: int, img_size: int, batch_shape) -> Placement:
    """LoadImagesAndLabels without augmentation (val.py's loader): load_image_label's resize to img_size (INTER_AREA when
    shrinking), then letterbox(img, batch_shape, auto=False, scaleup=False)."""
    (h, w), interp, r = load_image_size(h0, w0, img_size)
    if h < 1 or w < 1:
        raise RuntimeError(f"a {h0} x {w0} image resized to {img_size} has no pixels left ({h} x {w})")
    Hp, Wp = int(batch_shape[0]), int(batch_shape[1])
    (nw, nh), (top, bottom, left, right), ratio, pad = letterbox_geometry((h, w), (Hp, Wp), False, False, False)
    if (nw, nh) != (w, h):
        # the reference would resample the resized image a second time; rect_batch_shapes never makes a batch shape
        # smaller than one of its images, so this is reached only with a batch shape from elsewhere
        raise RuntimeError(f"batch shape {(Hp, Wp)} is smaller than the {h} x {w} image: it would be resampled twice")
    if (nh + top + bottom, nw + left + right) != (Hp, Wp):
        raise RuntimeError(f"letterbox of {h} x {w} into {(Hp, Wp)} does not fill it")
    return Placement(h0, w0, h, w, top, left, interp or LINEAR, ratio, pad, r, (h, w))


def place_from_shapes(entry) -> Tuple[Placement, Tuple[int, int]]:
    """The placement a rect loader's `shapes` entry ((h0, w0), ((h / h0, w / w0), (dw, dh))) describes (utils/datasets.py:590)
    -> (Placement, (Hp, Wp)): the resized h x w image (INTER_AREA when it shrank, as load_image_label chooses) under
    letterbox's border, top = round(dh - 0.1), left = round(dw - 0.1)."""
    (h0, w0), ((rh, rw), (dw, dh)) = entry
    h0, w0 = int(h0), int(w0)
    if h0 < 1 or w0 < 1:
        raise RuntimeError(f"empty image {(h0, w0)}")
    h, w = int(round(h0 * rh)), int(round(w0 * rw))
    if h < 1 or w < 1 or dw < 0 or dh < 0:
        raise RuntimeError(f"shapes entry {entry} leaves no image")
    interp = AREA if (h < h0 or w < w0) else LINEAR
    p = Placement(h0, w0, h, w, int(round(dh - 0.1)), int(round(dw - 0.1)), interp, (1.0, 1.0), (dw, dh),
                  max(h, w) / max(h0, w0), (h, w))
    return p, (int(round(h + 2 * dh)), int(round(w + 2 * dw)))


# ------------------------------------------------------------------------------------------------------ coefficient tables
def _scale(src: int, dst: int) -> float:
    return 1.0 / (dst / float(src))   # cv::resize: inv_scale = dsize / (double)ssize, scale = 1. / inv_scale


def _int_scale(scale: float) -> Optional[int]:
    k = int(np.rint(scale))
    return k if abs(scale - k) < _DBL_EPSILON else None


@functools.lru_cache(maxsize=256)
def _linear_table(src: int, dst: int, columns: bool) -> np.ndarray:
    """int32 [dst, 2]: first source index, coefficient pair (low | high << 16) of cv2's 8-bit INTER_LINEAR.  Columns outside
    the image move to the border pixel with fraction 0; rows keep their fraction (the kernel clips the two row indices)."""
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * _scale(src, dst) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if columns:
        lo, hi = s < 0, s >= src - 1
        f[lo | hi] = 0
        s[lo] = 0
        s[hi] = src - 1
    c0 = np.rint((np.float32(1.0) - f) * np.float32(2048)).astype(np.int64)   # saturate_cast<short>: round half to even
    c1 = np.rint(f * np.float32(2048)).astype(np.int64)
    out = np.stack([s, (c0 & 0xFFFF) | (c1 << 16)], 1).astype(np.int32)
    out.setflags(write=False)
    return out


@functools.lru_cache(maxsize=256)
def _area_table(src: int, dst: int) -> np.ndarray:
    """computeResizeAreaTab as int32 words: [dst + 1] first-tap indices, then per tap (source index, fp32 weight bits)."""
    scale = _scale(src, dst)
    f1 = np.arange(dst, dtype=np.float64) * scale
    f2 = f1 + scale
    cell = np.minimum(scale, src - f1)
    s2 = np.minimum(np.floor(f2).astype(np.int64), src - 1)
    s1 = np.minimum(np.ceil(f1).astype(np.int64), s2)
    head, tail = (s1 - f1) > 1e-3, (f2 - s2) > 1e-3
    mid = s2 - s1
    first = np.concatenate([[0], np.cumsum(head + mid + tail)])
    n = int(first[-1])
    si = np.empty(n, np.int64)
    al = np.empty(n, np.float32)
    si[first[:-1][head]] = s1[head] - 1
    al[first[:-1][head]] = ((s1 - f1) / cell)[head].astype(np.float32)
    k = np.arange(int(mid.sum())) - np.repeat(np.cumsum(mid) - mid, mid)
    pos = np.repeat(first[:-1] + head, mid) + k
    si[pos] = np.repeat(s1, mid) + k
    al[pos] = np.repeat((1.0 / cell).astype(np.float32), mid)
    si[first[1:][tail] - 1] = s2[tail]
    al[first[1:][tail] - 1] = (np.minimum(np.minimum(f2 - s2, 1.0), cell) / cell)[tail].astype(np.float32)
    taps = np.stack([si.astype(np.int32), al.view(np.int32)], 1).reshape(-1)
    out = np.concatenate([first.astype(np.int32), taps])
    out.setflags(write=False)
    return out


def resample_plan(h0: int, w0: int, new_h: int, new_w: int, interp: str):
    """How cv2.resize(img, (new_w, new_h), interpolation=interp) resamples a uint8 h0 x w0 image:
    -> (mode, kx, ky, inv_area fp32, column table, row table) for y5obb_letterbox_s2d_u8."""
    none = np.zeros(0, np.int32)
    if interp not in (LINEAR, AREA):
        raise RuntimeError(f"interpolation must be '{LINEAR}' or '{AREA}', got {interp!r}")
    if (new_h, new_w) == (h0, w0):
        return MODE_COPY, 0, 0, np.float32(0), none, none
    kx, ky = _int_scale(_scale(w0, new_w)), _int_scale(_scale(h0, new_h))
    if interp == LINEAR and not (kx == 2 and ky == 2):   # (exactly 2 x 2: cv2 resamples INTER_LINEAR as INTER_AREA)
        return MODE_LINEAR, 0, 0, np.float32(0), _linear_table(w0, new_w, True).reshape(-1), \
            _linear_table(h0, new_h, False).reshape(-1)
    if new_h > h0 or new_w > w0:
        raise RuntimeError(f"INTER_AREA enlargement ({h0} x {w0} -> {new_h} x {new_w}) is not covered: the reference only "
                           "shrinks with it")
    if kx is not None and ky is not None:
        return MODE_AREA_INT, kx, ky, np.float32(1.0) / np.float32(kx * ky), none, none
    return MODE_AREA, 0, 0, np.float32(0), _area_table(w0, new_w), _area_table(h0, new_h)


# ------------------------------------------------------------------------------------------------------------------ packing
def as_image(im) -> np.ndarray:
    """A decoded image (numpy array or CPU tensor) as contiguous uint8 [H, W, 3]; anything else is refused."""
    if isinstance(im, torch.Tensor):
        if im.is_cuda:
            raise RuntimeError("source images are host arrays (as cv2.imread returns them)")
        im = im.numpy()
    if not isinstance(im, np.ndarray) or im.dtype != np.uint8:
        raise RuntimeError(f"an image must be a uint8 array, got {getattr(im, 'dtype', type(im))}")
    if im.ndim != 3 or im.shape[2] != 3:
        raise RuntimeError(f"an image must be [H, W, 3] (BGR), got {tuple(im.shape)}")
    if im.shape[0] < 1 or im.shape[1] < 1:
        raise RuntimeError(f"empty image {tuple(im.shape)}")
    return np.ascontiguousarray(im)


class PackedBatch:
    """One pinned host buffer holding a batch for y5obb_letterbox_s2d_u8: B descriptors, the coefficient tables, the
    per-image (pad_x, pad_y, gain) of scale_polys, then the source images back to back.  One copy uploads all of it."""

    def __init__(self, host: torch.Tensor, nbytes: int, B: int, Hp: int, Wp: int, desc_bytes: int, pad_gain_off: int,
                 src_off: int, src_bytes: int):
        self.host, self.nbytes, self.B, self.Hp, self.Wp = host, nbytes, B, Hp, Wp
        self.desc_bytes, self.pad_gain_off, self.src_off, self.src_bytes = desc_bytes, pad_gain_off, src_off, src_bytes


def packed_bytes(images: Sequence[np.ndarray], plans) -> Tuple[int, int, int]:
    """(descriptor + table bytes, offset of the source images, total bytes) of a batch."""
    words = DESC_WORDS * len(images) + sum(p[4].size + (p[4].size & 1) + p[5].size + (p[5].size & 1) for p in plans)
    words += 3 * len(images)
    src_off = (words * 4 + 255) // 256 * 256
    return words * 4, src_off, src_off + sum(int(im.size) for im in images)


def pack_batch(images: Sequence[np.ndarray], placements: Sequence[Placement], Hp: int, Wp: int,
               host: Optional[torch.Tensor] = None) -> PackedBatch:
    """images: as_image() arrays; placements: one Placement each.  `host`: a pinned uint8 tensor to fill (a new one is
    allocated when it is missing or too small)."""
    B = len(images)
    if B == 0 or B != len(placements):
        raise RuntimeError("pack_batch wants one placement per image and at least one image")
    plans = [resample_plan(p.h0, p.w0, p.new_h, p.new_w, p.interp) for p in placements]
    desc_bytes, src_off, total = packed_bytes(images, plans)
    if host is None or host.numel() < total:
        host = torch.empty(int(total * 1.25) + 4096, dtype=torch.uint8)
        if torch.cuda.is_available():   # (the layout itself needs no device: tests read it back on the CPU)
            host = host.pin_memory()
    buf = host.numpy()
    w32 = buf[:desc_bytes].view(np.int32)
    f32 = buf[:desc_bytes].view(np.float32)
    off = DESC_WORDS * B
    src = src_off
    for b, (im, p, (mode, kx, ky, inv_area, xt, yt)) in enumerate(zip(images, placements, plans)):
        if tuple(im.shape[:2]) != (p.h0, p.w0):
            raise RuntimeError(f"image {b} is {tuple(im.shape[:2])}, its placement was made for {(p.h0, p.w0)}")
        d = w32[DESC_WORDS * b:DESC_WORDS * (b + 1)]
        d[:] = 0
        d[0:2].view(np.int64)[0] = src - src_off
        d[2:11] = (p.h0, p.w0, p.new_h, p.new_w, p.top, p.left, mode, kx, ky)
        f32[DESC_WORDS * b + 11] = inv_area
        for slot, t in ((12, xt), (13, yt)):
            d[slot] = off
            w32[off:off + t.size] = t
            off += t.size + (t.size & 1)
        buf[src:src + im.size] = im.reshape(-1)
        src += im.size
    pad_gain_off = off
    for p in placements:
        f32[off:off + 3] = p.pad_gain
        off += 3
    return PackedBatch(host, total, B, Hp, Wp, desc_bytes, pad_gain_off * 4, src_off, src - src_off)


def letterbox_s2d(dev_buf: torch.Tensor, batch: PackedBatch, x_s2d: torch.Tensor, pad_cols: int = 1) -> None:
    """Launches y5obb_letterbox_s2d_u8 (_f16) on the current stream: dev_buf holds batch.host[:batch.nbytes] on the device,
    x_s2d [B, Hp/2, Wp/2 + 2*pad_cols, 16] bf16 (fp16) is the plan's stem input."""
    _lib.require_cuda(dev_buf, "dev_buf")
    want = (batch.B, batch.Hp // 2, batch.Wp // 2 + 2 * pad_cols, 16)
    if x_s2d.dtype not in (torch.bfloat16, torch.float16) or tuple(x_s2d.shape) != want or not x_s2d.is_contiguous():
        raise RuntimeError(f"x_s2d must be contiguous bf16 or fp16 {want}, got {x_s2d.dtype} {tuple(x_s2d.shape)}")
    name = "y5obb_letterbox_s2d_u8" + ("_f16" if x_s2d.dtype == torch.float16 else "")
    if dev_buf.dtype != torch.uint8 or dev_buf.numel() < batch.nbytes:
        raise RuntimeError("dev_buf is smaller than the packed batch")
    base = dev_buf.data_ptr()
    with torch.cuda.device(dev_buf.device):
        _lib.check(getattr(_lib.lib(), name)(base + batch.src_off, batch.src_bytes, base, batch.host.data_ptr(),
                                             batch.desc_bytes, batch.B, batch.Hp, batch.Wp, x_s2d.data_ptr(), pad_cols,
                                             _lib.stream_ptr(dev_buf.device)), name)


def letterboxed_records(model, dev_buf: torch.Tensor, batch: PackedBatch, device, slot: int = 0):
    """Runs a packed batch through `model`'s records plan for the batch's shape and `slot`, on the current stream:
    letterbox_s2d writes the plan's stem input from dev_buf (batch.host[:batch.nbytes] on the device), then forward_s2d.
    -> (general.DetectRecords, the per-image (pad_x, pad_y, gain) fp32 table for scale_polys_batched, a view of dev_buf)."""
    eng = model.records_plan((batch.B, 3, batch.Hp, batch.Wp), device, slot)
    letterbox_s2d(dev_buf, batch, eng.x_s2d, 1)
    pad_gain = dev_buf[batch.pad_gain_off:batch.pad_gain_off + 12 * batch.B].view(torch.float32)
    return DetectRecords(eng.forward_s2d(), eng.nc, eng.half), pad_gain


def scale_polys_batched(rows: torch.Tensor, counts: torch.Tensor, pad_gain: torch.Tensor) -> torch.Tensor:
    """rbox2poly then scale_polys for a batch's packed NMS output in one launch: rows [B, max_det, 7] fp32, counts int64
    [>= B], pad_gain [B, 3] fp32 (pad_x, pad_y, gain) per image -> polys [B, max_det, 8] in source pixels (rows >= counts[b]
    are zero).  Equal to rboxs_utils.rbox2poly + scale_polys per image, bit for bit."""
    for t, name in ((rows, "rows"), (counts, "counts"), (pad_gain, "pad_gain")):
        _lib.require_cuda(t, name)
    B, max_det = rows.shape[0], rows.shape[1]
    if rows.dtype != torch.float32 or rows.dim() != 3 or rows.shape[2] != 7 or counts.dtype != torch.int64 or \
            counts.numel() < B or pad_gain.dtype != torch.float32 or pad_gain.numel() != 3 * B:
        raise RuntimeError("scale_polys_batched wants rows fp32 [B, max_det, 7], counts int64 [>= B], pad_gain fp32 [B, 3]")
    rows, counts, pad_gain = rows.contiguous(), counts.contiguous(), pad_gain.contiguous()
    polys = torch.empty((B, max_det, 8), dtype=torch.float32, device=rows.device)
    with torch.cuda.device(rows.device):
        _lib.check(_lib.lib().y5obb_scale_polys_batched_f32(rows.data_ptr(), counts.data_ptr(), pad_gain.data_ptr(), B, max_det,
                                                            polys.data_ptr(), _lib.stream_ptr(rows.device)),
                   "y5obb_scale_polys_batched_f32")
    return polys


def detect_pad_gain(img1_shape, img0_shape) -> Tuple[float, float, float]:
    """(pad_x, pad_y, gain) as scale_polys forms them from the two shapes when ratio_pad is None (detect.py:147,
    utils/general.py:638-640)."""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    return (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2, gain
