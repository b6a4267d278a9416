"""numpy restatement of the reference's training augmentation arithmetic (utils/datasets.py:561-665,
utils/augmentations.py), per sample, from a host plan of yolov5_obb_b200.augment.  Test infrastructure only: the device
path is csrc/augment.cu.  tests/test_augment_cpu.py pins each piece to cv2 where cv2 imports.

  warp_affine_u8   cv2.warpAffine, 8UC3, INTER_LINEAR, BORDER_CONSTANT 114: fixed point with AB_BITS = 10, INTER_BITS = 5,
                   bilinear weights of the 32 x 32 table (exact products of 1/32 steps, scaled to 2^15), (sum + 2^14) >> 15
  bgr2hsv_u8       cv2.COLOR_BGR2HSV, 8U: the 12-bit division tables
  hsv2bgr_u8       cv2.COLOR_HSV2BGR, 8U (OpenCV 4.13, the vector loop that converts rows in blocks of 4 SIMD
                   widths): fp32 sector formula, 1 - s*f as one fused multiply-add, trunc(x * 255)
  sample_image     one augmented image (HWC BGR uint8) of a plan record: virtual canvas, warp, mixup, HSV, flips
  sample_polys     the fp32 [n, 9] (cls, poly) labels of a plan record before poly2rbox, in the reference's order
"""
import numpy as np

BORDER = 114
AB_BITS, INTER_BITS = 10, 5


def canvas(group, images, side):
    """The canvas a warp samples: the 2S mosaic of load_mosaic (:725-786) or the letterboxed image, over 114."""
    c = np.full((side, side, 3), BORDER, np.uint8)
    for img_id, (x1a, y1a, x2a, y2a), (pw, ph) in zip(group["img"], group["rect"], group["pad"]):
        c[y1a:y2a, x1a:x2a] = images[img_id][y1a - ph:y2a - ph, x1a - pw:x2a - pw]
    return c


def warp_affine_u8(src, minv, out_w, out_h):
    """cv2.warpAffine(src, M, (out_w, out_h), borderValue=(114,)*3) with minv = the inverse of M as warpAffine computes it."""
    m0, m1, m2, m3, m4, m5 = (float(v) for v in minv)
    x = np.arange(out_w, dtype=np.float64)
    y = np.arange(out_h, dtype=np.float64)
    sc = float(1 << AB_BITS)
    rd = (1 << AB_BITS) >> INTER_BITS >> 1
    adelta = np.rint(m0 * x * sc).astype(np.int64)
    bdelta = np.rint(m3 * x * sc).astype(np.int64)
    X0 = np.rint((m1 * y + m2) * sc).astype(np.int64) + rd
    Y0 = np.rint((m4 * y + m5) * sc).astype(np.int64) + rd
    X = (X0[:, None] + adelta[None, :]) >> (AB_BITS - INTER_BITS)
    Y = (Y0[:, None] + bdelta[None, :]) >> (AB_BITS - INTER_BITS)
    ix, iy = X >> INTER_BITS, Y >> INTER_BITS
    fx, fy = X & 31, Y & 31
    h, w = src.shape[:2]
    acc = np.zeros((out_h, out_w, 3), np.int64)
    for dy, wy in ((0, 32 - fy), (1, fy)):
        for dx, wx in ((0, 32 - fx), (1, fx)):
            sx, sy = ix + dx, iy + dy
            ok = (sx >= 0) & (sx < w) & (sy >= 0) & (sy < h)
            p = np.where(ok[..., None], src[np.clip(sy, 0, h - 1), np.clip(sx, 0, w - 1)], BORDER).astype(np.int64)
            acc += p * (wy * wx * 32)[..., None]
    return ((acc + (1 << 14)) >> 15).astype(np.uint8)


def bgr2hsv_u8(img):
    sh = 12
    i = np.arange(256, dtype=np.float64)
    with np.errstate(divide="ignore"):
        sdiv = np.where(i > 0, np.rint((255 << sh) / i), 0).astype(np.int64)
        hdiv = np.where(i > 0, np.rint((180 << sh) / (6.0 * i)), 0).astype(np.int64)
    b, g, r = (img[..., k].astype(np.int64) for k in range(3))
    v = np.maximum(np.maximum(b, g), r)
    vmin = np.minimum(np.minimum(b, g), r)
    diff = v - vmin
    s = (diff * sdiv[v] + (1 << (sh - 1))) >> sh
    h = np.where(v == r, g - b, np.where(v == g, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * hdiv[diff] + (1 << (sh - 1))) >> sh
    h = h + np.where(h < 0, 180, 0)
    return np.stack([h, s, v], -1).astype(np.uint8)


_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def _fma_f32(a, b, c):  # a*b + c with one rounding to fp32 (the fp64 product of two fp32 values is exact)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def hsv2bgr_u8(hsv):
    f32 = np.float32
    h = hsv[..., 0].astype(f32) * f32(6.0 / 180.0)
    sec = np.floor(h)
    f = (h - sec).astype(f32)
    sec = sec.astype(np.int64) % 6
    s = hsv[..., 1].astype(f32) * f32(1.0 / 255.0)
    v = hsv[..., 2].astype(f32) * f32(1.0 / 255.0)
    one = np.ones_like(s)
    tab = [v, v * (one - s), v * _fma_f32(-s, f, one), v * _fma_f32(-s, one - f, one)]
    out = [np.choose(_SECTOR[sec, k], tab) for k in range(3)]
    return np.stack([np.trunc(o * f32(255.0)) for o in out], -1).astype(np.uint8)


def sample_image(rec, images, S):
    """One augmented sample, HWC BGR uint8 before the CHW / RGB transpose of __getitem__."""
    out = []
    for g in rec["groups"]:
        c = canvas(g, images, g["canvas"])
        out.append(warp_affine_u8(c, g["minv"], S, S))
    img = out[0]
    if rec["mix_r"] is not None:   # mixup (utils/augmentations.py:276-281)
        img = (img * rec["mix_r"] + out[1] * (1 - rec["mix_r"])).astype(np.uint8)
    if rec["luts"] is not None:    # augment_hsv (:48-61)
        hsv = bgr2hsv_u8(img)
        hsv = np.stack([rec["luts"][k][hsv[..., k]] for k in range(3)], -1)
        img = hsv2bgr_u8(hsv)
    if rec["flipud"]:
        img = img[::-1]
    if rec["fliplr"]:
        img = img[:, ::-1]
    return np.ascontiguousarray(img)


def _poly_filter(polys, h, w):  # utils/rboxs_utils.py:183-199, in the dtype of polys
    x, y = polys[:, 0::2], polys[:, 1::2]
    xc = (x.max(1) + x.min(1)) / 2.0
    yc = (y.max(1) + y.min(1)) / 2.0
    return (xc > 0) & (xc < w) & (yc > 0) & (yc < h)


def sample_polys(rec, labels, S):
    """fp32 [n, 9] (cls, poly) after pads, poly_filter, the affine map, mixup concatenation and flips."""
    parts = []
    for g in rec["groups"]:
        lab = []
        for img_id, (lw, lh) in zip(g["img"], g["lpad"]):
            L = labels[img_id].copy()
            L[:, 1::2] = L[:, 1::2] + np.float32(lw)
            L[:, 2::2] = L[:, 2::2] + np.float32(lh)
            lab.append(L)
        L = np.concatenate(lab, 0) if lab else np.zeros((0, 9), np.float32)
        if g["canvas"] != S:   # load_mosaic's filter on the 2S canvas, fp32
            L = L[_poly_filter(L[:, 1:].copy(), g["canvas"], g["canvas"])]
        if len(L):
            M = g["M"]
            xy = np.ones((len(L) * 4, 3))
            xy[:, :2] = L[:, 1:].reshape(-1, 2)
            xy = (xy @ M.T)[:, :2].reshape(-1, 8)
            keep = _poly_filter(xy, S, S)
            L[:, 1:] = xy
            L = L[keep]
        parts.append(L)
    L = np.concatenate(parts, 0)
    if rec["flipud"] and len(L):
        L[:, 2::2] = S - L[:, 2::2] - 1
    if rec["fliplr"] and len(L):
        L[:, 1::2] = S - L[:, 1::2] - 1
    return L


def targets_from_polys(L, S, nc_theta=180, radius=2.0):
    """The rows of __getitem__ (:637-659) from fp32 polys, with the restated poly2rbox: [n, 186] (cls, rbox, csl)."""
    from oracle import rbox_ref
    if not len(L):
        return np.zeros((0, 6 + nc_theta), np.float32)
    rb = rbox_ref.poly2rbox(L[:, 1:], use_pi=True)
    angle = rb[:, 4] * 180 / rbox_ref.PI_REF + 90
    x = np.arange(-nc_theta / 2, nc_theta / 2)
    ysig = np.exp(-(x ** 2) / (2 * radius ** 2))
    csl = np.stack([np.roll(ysig, -int(nc_theta / 2 - a)) for a in angle])
    rows = np.concatenate([L[:, :1], rb, csl], 1)
    mask = (rb[:, 0] >= 0) & (rb[:, 0] < S) & (rb[:, 1] >= 0) & (rb[:, 0] < S) & (rb[:, 2] > 5) | (rb[:, 3] > 5)
    return rows[mask].astype(np.float32)
