"""Training augmentation on the device: what LoadImagesAndLabels.__getitem__ + collate_fn (utils/datasets.py:561-672) do
for a batch, in two launches and one scan (csrc/augment.cu).

    plan_sample(...)      the only per-sample Python: the reference's random draws in its order, and the numbers they
                          make (placements, the fp64 affine matrix and its inverse, mixup ratio, HSV LUTs, flips).
                          It touches no pixel.
    DeviceDataset         the cached dataset on the device (images as load_image_label returns them, labels [n, 9])
    augment_batch(...)    one batch on the device: uint8 [B, 3, S, S] RGB images and [nt, 187] (or [nt, 8]) targets
    DeviceAugmentLoader   the iterable train.py's loop consumes: `for imgs, tg in loader: ts.step(imgs, tg)`

Scope: the training branch of __getitem__ (augment=True, rect=False) with perspective == 0.  Images are cached with their
longest side equal to img_size (what --cache ram stores), so letterbox pads and never resizes.
"""
import ctypes
import math
import random
from ctypes import c_int

import numpy as np
import torch

from . import _lib

BORDER = 114
MAX_PLACE = 8           # 4 mosaic placements per group, two groups (the second one is mixup's mosaic)
F_MOSAIC, F_MIXUP, F_HSV, F_FLIPUD, F_FLIPLR = 1, 2, 4, 8, 16


class SampleRec(ctypes.Structure):
    """y5obb_augment_sample of include/y5obb.h."""
    _fields_ = [("img", c_int * MAX_PLACE), ("rect", c_int * (4 * MAX_PLACE)), ("pad", c_int * (2 * MAX_PLACE)),
                ("lpad", ctypes.c_float * (2 * MAX_PLACE)), ("minv", ctypes.c_double * 12), ("m", ctypes.c_double * 12),
                ("mix_r", ctypes.c_double), ("mix_1mr", ctypes.c_double), ("n_place", c_int * 2), ("canvas", c_int * 2),
                ("flags", c_int), ("reserved", c_int), ("lut", ctypes.c_uint8 * 768)]


def rotation_matrix_2d(angle, scale):
    """cv2.getRotationMatrix2D(angle=angle, center=(0, 0), scale=scale), in its arithmetic."""
    a = angle * (math.pi / 180)
    alpha = math.cos(a) * scale
    beta = math.sin(a) * scale
    cx = cy = 0.0
    return np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]])


def invert_affine(M):
    """The inverse warpAffine computes from a 2 x 3 matrix (cv2.invertAffineTransform's order), as 6 doubles."""
    m = [float(v) for v in np.asarray(M, np.float64).reshape(-1)[:6]]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22 = m[4] * D, m[0] * D
    m[0], m[1], m[3], m[4] = a11, m[1] * -D, m[3] * -D, a22
    b1 = -m[0] * m[2] - m[1] * m[5]
    b2 = -m[3] * m[2] - m[4] * m[5]
    m[2], m[5] = b1, b2
    return np.array(m)


def _perspective_matrix(hyp, width, height, shape_hw):
    """random_perspective's eight draws and M = T @ S @ R @ P @ C (utils/augmentations.py:131-168)."""
    if hyp["perspective"]:
        raise ValueError("perspective != 0 (cv2.warpPerspective) is not supported by the device augmentation")
    C = np.eye(3)
    C[0, 2] = -shape_hw[1] / 2
    C[1, 2] = -shape_hw[0] / 2
    P = np.eye(3)
    P[2, 0] = random.uniform(-hyp["perspective"], hyp["perspective"])
    P[2, 1] = random.uniform(-hyp["perspective"], hyp["perspective"])
    R = np.eye(3)
    a = random.uniform(-hyp["degrees"], hyp["degrees"])
    s = random.uniform(1 - hyp["scale"], 1 + hyp["scale"])
    R[:2] = rotation_matrix_2d(a, s)
    S = np.eye(3)
    S[0, 1] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    S[1, 0] = math.tan(random.uniform(-hyp["shear"], hyp["shear"]) * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * width
    T[1, 2] = random.uniform(0.5 - hyp["translate"], 0.5 + hyp["translate"]) * height
    return T @ S @ R @ P @ C


def _mosaic_group(index, n, shapes, S, hyp):
    """load_mosaic (utils/datasets.py:725-786): centre, 3 extra images, shuffle, placements, then random_perspective with
    border -S/2.  copy_paste (:777) makes no random call and changes nothing: OBB segments are always empty."""
    yc, xc = (int(random.uniform(-x, 2 * S + x)) for x in (-S // 2, -S // 2))
    indices = [index] + random.choices(range(n), k=3)
    random.shuffle(indices)
    rect, pad = [], []
    for i, idx in enumerate(indices):
        h, w = shapes[idx]
        if i == 0:
            x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
            x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
        elif i == 1:
            x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, S * 2), yc
            x1b, y1b = 0, h - (y2a - y1a)
        elif i == 2:
            x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(S * 2, yc + h)
            x1b, y1b = w - (x2a - x1a), 0
        else:
            x1a, y1a, x2a, y2a = xc, yc, min(xc + w, S * 2), min(S * 2, yc + h)
            x1b, y1b = 0, 0
        rect.append((x1a, y1a, x2a, y2a))
        pad.append((x1a - x1b, y1a - y1b))
    side = 2 * S
    M = _perspective_matrix(hyp, side + 2 * (-S // 2), side + 2 * (-S // 2), (side, side))
    return dict(img=indices, rect=rect, pad=pad, lpad=[(float(a), float(b)) for a, b in pad], canvas=side, M=M,
                minv=invert_affine(M[:2]))


def _letterbox_group(index, shapes, S, hyp):
    """load_image_label + letterbox(auto=False) + random_perspective with border 0 (utils/datasets.py:585-604).  The
    cached image's longest side is S, so letterbox only pads: the image goes at (round(dw - 0.1), round(dh - 0.1)) and the
    labels move by (dw, dh)."""
    h, w = shapes[index]
    dw, dh = (S - w) / 2, (S - h) / 2
    top, left = int(round(dh - 0.1)), int(round(dw - 0.1))
    M = _perspective_matrix(hyp, S, S, (S, S))
    return dict(img=[index], rect=[(left, top, left + w, top + h)], pad=[(left, top)], lpad=[(dw, dh)], canvas=S, M=M,
                minv=invert_affine(M[:2]))


def plan_sample(index, n, shapes, S, hyp):
    """The random draws of one __getitem__(index) (utils/datasets.py:561-633) on the module-level `random` and `np.random`
    generators, in the reference's order, and the record the device needs for them."""
    groups, mix_r = [], None
    if random.random() < hyp["mosaic"]:
        groups.append(_mosaic_group(index, n, shapes, S, hyp))
        if random.random() < hyp["mixup"]:
            groups.append(_mosaic_group(random.randint(0, n - 1), n, shapes, S, hyp))
            mix_r = np.random.beta(32.0, 32.0)
    else:
        groups.append(_letterbox_group(index, shapes, S, hyp))
    luts = None
    hg, sg, vg = hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]
    if hg or sg or vg:   # augment_hsv (utils/augmentations.py:48-61)
        r = np.random.uniform(-1, 1, 3) * [hg, sg, vg] + 1
        x = np.arange(0, 256, dtype=r.dtype)
        luts = np.stack([((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
                         np.clip(x * r[2], 0, 255).astype(np.uint8)])
    flipud = random.random() < hyp["flipud"]
    fliplr = random.random() < hyp["fliplr"]
    return dict(groups=groups, mix_r=mix_r, luts=luts, flipud=flipud, fliplr=fliplr)


def pack_record(rec):
    """A plan record as the device's y5obb_augment_sample."""
    r = SampleRec()
    flags = 0
    for g, grp in enumerate(rec["groups"]):
        r.n_place[g] = len(grp["img"])
        r.canvas[g] = grp["canvas"]
        for i in range(len(grp["img"])):
            p = 4 * g + i
            r.img[p] = grp["img"][i]
            r.rect[4 * p:4 * p + 4] = grp["rect"][i]
            r.pad[2 * p:2 * p + 2] = grp["pad"][i]
            r.lpad[2 * p:2 * p + 2] = grp["lpad"][i]
        r.minv[6 * g:6 * g + 6] = [float(v) for v in grp["minv"]]
        r.m[6 * g:6 * g + 6] = [float(v) for v in grp["M"][:2].reshape(-1)]
    if len(rec["groups"][0]["img"]) == 4:
        flags |= F_MOSAIC
    if rec["mix_r"] is not None:
        flags |= F_MIXUP
        r.mix_r, r.mix_1mr = float(rec["mix_r"]), float(1 - rec["mix_r"])
    if rec["luts"] is not None:
        flags |= F_HSV
        ctypes.memmove(r.lut, np.ascontiguousarray(rec["luts"], np.uint8).ctypes.data, 768)
    flags |= F_FLIPUD if rec["flipud"] else 0
    flags |= F_FLIPLR if rec["fliplr"] else 0
    r.flags = flags
    return r


class DeviceDataset:
    """The training set held on the device: images uint8 BGR HWC with their longest side == img_size (load_image_label's
    cached form, utils/datasets.py:702-722) and labels [n_i, 9] fp32 (cls, poly) rows (verify_image_label's form), each in
    one flat buffer with 64-bit offsets."""

    def __init__(self, images, labels, img_size, device="cuda"):
        S = int(img_size)
        if S <= 0 or S % 32:
            raise ValueError(f"img_size must be a positive multiple of 32, got {img_size}")
        if len(images) != len(labels) or not len(images):
            raise ValueError("images and labels must be non-empty lists of the same length")
        shapes, ioff, loff, lcnt = [], [0], [0], []
        for k, (im, lb) in enumerate(zip(images, labels)):
            im = np.asarray(im)
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"image {k}: expected uint8 HWC BGR, got {im.dtype} {im.shape}")
            if max(im.shape[:2]) != S:
                raise ValueError(f"image {k}: longest side {max(im.shape[:2])} != img_size {S} (resize when caching)")
            lb = np.asarray(lb, np.float32).reshape(-1, 9)
            shapes.append(im.shape[:2])
            ioff.append(ioff[-1] + im.size)
            loff.append(loff[-1] + lb.shape[0])
            lcnt.append(lb.shape[0])
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device, self.img_size, self.n = dev, S, len(images)
        self.shapes = shapes
        self.label_counts = np.array(lcnt, np.int64)
        self.images = torch.from_numpy(np.concatenate([np.asarray(im).reshape(-1) for im in images])).to(dev)
        self.labels = torch.from_numpy(np.concatenate([np.asarray(lb, np.float32).reshape(-1, 9) for lb in labels]
                                                      ).reshape(-1)).to(dev)
        hw = np.array(shapes, np.int32).reshape(-1, 2)
        self.meta_host = np.ascontiguousarray(np.stack([np.array(ioff[:-1], np.int64), hw[:, 0].astype(np.int64),
                                                        hw[:, 1].astype(np.int64), np.array(loff[:-1], np.int64),
                                                        self.label_counts], 1))
        self.img_meta = torch.from_numpy(self.meta_host.reshape(-1).copy()).to(dev)

    def __len__(self):
        return self.n


def plan_batch(dataset, indices, hyp):
    return [plan_sample(int(i), dataset.n, dataset.shapes, dataset.img_size, hyp) for i in indices]


class _Staging:
    """Host and device buffers of one batch in flight; they grow and are reused."""

    def __init__(self):
        self.rec_h = self.rec_d = self.cand_h = self.cand_d = None
        self.nt_h = torch.empty(1, dtype=torch.int64).pin_memory()
        self.rows = self.imgs = self.ws = self.nt_d = None
        self.ready = torch.cuda.Event()


def _grow(t, n, dtype, device, pinned=False):
    if t is not None and t.numel() >= n:
        return t
    t = torch.empty(max(int(n * 1.25), 64), dtype=dtype, device=device)
    return t.pin_memory() if pinned else t


def launch_batch(dataset, recs, tcols=187, nc_theta=180, csl_radius=2.0, stage=None, stream=None):
    """Enqueue one batch on `stream` (default: the current stream).  Returns (imgs [B,3,S,S] uint8, rows, stage), where the
    first nt rows of `rows` are the targets; nt lands in stage.nt_h once stage.ready has completed."""
    if tcols not in (8, 7 + nc_theta):
        raise ValueError("tcols must be 187 (7 + cls_theta, the reference's rows) or 8 (compact rows)")
    dev, S = dataset.device, dataset.img_size
    B = len(recs)
    if B == 0:
        raise ValueError("empty batch")
    stage = stage or _Staging()
    st = torch.cuda.current_stream(dev) if stream is None else stream
    L = _lib.lib()
    rsz = ctypes.sizeof(SampleRec)
    stage.rec_h = _grow(stage.rec_h, B * rsz, torch.uint8, "cpu", pinned=True)
    packed = (SampleRec * B)(*[pack_record(r) for r in recs])
    _lib.check(L.y5obb_augment_check(dataset.meta_host.ctypes.data, dataset.n, dataset.images.numel(),
                                     dataset.labels.numel() // 9, ctypes.addressof(packed), B, S), "y5obb_augment_check")
    ctypes.memmove(stage.rec_h.data_ptr(), packed, B * rsz)
    # per-placement label ranges in (sample, group, placement) order: the reference's concatenation order
    counts = np.zeros(B * MAX_PLACE, np.int64)
    for b, r in enumerate(recs):
        for g, grp in enumerate(r["groups"]):
            for i, idx in enumerate(grp["img"]):
                counts[b * MAX_PLACE + 4 * g + i] = dataset.label_counts[idx]
    start = np.zeros(B * MAX_PLACE + 1, np.int64)
    np.cumsum(counts, out=start[1:])
    ncand = int(start[-1])
    stage.cand_h = _grow(stage.cand_h, B * MAX_PLACE + 1, torch.int64, "cpu", pinned=True)
    stage.cand_h[:B * MAX_PLACE + 1].numpy()[:] = start
    with torch.cuda.stream(st):
        stage.rec_d = _grow(stage.rec_d, B * rsz, torch.uint8, dev)
        stage.cand_d = _grow(stage.cand_d, B * MAX_PLACE + 1, torch.int64, dev)
        stage.rec_d[:B * rsz].copy_(stage.rec_h[:B * rsz], non_blocking=True)
        stage.cand_d[:B * MAX_PLACE + 1].copy_(stage.cand_h[:B * MAX_PLACE + 1], non_blocking=True)
        if stage.imgs is None or stage.imgs.shape != (B, 3, S, S):
            stage.imgs = torch.empty((B, 3, S, S), dtype=torch.uint8, device=dev)
        stage.rows = _grow(stage.rows, max(ncand, 1) * tcols, torch.float32, dev)
        stage.nt_d = _grow(stage.nt_d, 1, torch.int64, dev)
        wsb = L.y5obb_augment_labels_workspace_bytes(ncand)
        stage.ws = _grow(stage.ws, wsb, torch.uint8, dev)
        sp = st.cuda_stream
        _lib.check(L.y5obb_augment_images_u8(dataset.images.data_ptr(), dataset.img_meta.data_ptr(), dataset.n,
                                             stage.rec_d.data_ptr(), B, S, stage.imgs.data_ptr(), sp),
                   "y5obb_augment_images_u8")
        _lib.check(L.y5obb_augment_labels(dataset.labels.data_ptr(), dataset.img_meta.data_ptr(), dataset.n,
                                          stage.rec_d.data_ptr(), stage.cand_d.data_ptr(), B, ncand, S, nc_theta,
                                          float(csl_radius), tcols, stage.rows.data_ptr(), stage.nt_d.data_ptr(),
                                          stage.ws.data_ptr(), stage.ws.numel(), sp),
                   "y5obb_augment_labels")
        stage.nt_h.copy_(stage.nt_d[:1], non_blocking=True)
        stage.ready.record(st)
    return stage.imgs, stage.rows, stage


def augment_batch(dataset, recs, tcols=187, nc_theta=180, csl_radius=2.0):
    """One batch, blocking: (imgs uint8 [B,3,S,S] RGB, targets [nt, tcols] fp32) as collate_fn yields them."""
    imgs, rows, stage = launch_batch(dataset, recs, tcols, nc_theta, csl_radius)
    stage.ready.synchronize()
    nt = int(stage.nt_h.item())
    return imgs.clone(), rows[:nt * tcols].view(nt, tcols).clone()


class DeviceAugmentLoader:
    """The training DataLoader of utils/datasets.py:95-122 (augment=True, rect=False, one process) on the device.

    Batches of indices come from torch's own DataLoader machinery over the same sampler the reference builds (a repeating
    RandomSampler when shuffle), so they consume the same draws of torch's global generator; every sample then draws from
    `random` / `np.random` in __getitem__'s order.  seed: if given, seeds the three generators first (train.py's
    init_seeds).  Each yielded (imgs, targets) is built on a side stream while the caller's step on the previous batch runs;
    the current stream waits on an event, and the only host read (nt) is a pinned copy after the side stream's event.  The
    buffers are double-buffered: a yielded batch stays valid until the batch after the next one is requested."""

    def __init__(self, dataset, hyp, batch_size, shuffle=True, seed=None, compact=False):
        for k in ("mosaic", "mixup", "degrees", "translate", "scale", "shear", "perspective", "hsv_h", "hsv_s", "hsv_v",
                  "flipud", "fliplr"):
            if k not in hyp:
                raise KeyError(f"hyp lacks '{k}'")
        if hyp["perspective"]:
            raise ValueError("perspective != 0 (cv2.warpPerspective) is not supported by the device augmentation")
        self.dataset, self.hyp, self.batch_size = dataset, dict(hyp), int(batch_size)
        self.nc_theta = int(hyp.get("cls_theta", 180))
        self.radius = float(hyp.get("csl_radius", 6.0))
        self.tcols = 8 if compact else 7 + self.nc_theta
        if seed is not None:
            random.seed(seed)
            np.random.seed(seed)
            torch.manual_seed(seed)
        from torch.utils.data import BatchSampler, DataLoader, RandomSampler, SequentialSampler
        base = RandomSampler(range(dataset.n)) if shuffle else SequentialSampler(range(dataset.n))
        self._batches = BatchSampler(base, self.batch_size, drop_last=False)

        class _Repeat:
            def __init__(s, bs):
                s.bs = bs

            def __iter__(s):
                while True:
                    yield from iter(s.bs)

        self._it = iter(DataLoader(range(dataset.n), batch_sampler=_Repeat(self._batches), collate_fn=list, num_workers=0))
        self._stream = torch.cuda.Stream(dataset.device)
        self._stages = [_Staging(), _Staging()]
        self._consumed = [torch.cuda.Event(), torch.cuda.Event()]

    def __len__(self):
        return len(self._batches)

    def _launch(self, j):
        recs = plan_batch(self.dataset, next(self._it), self.hyp)
        s = self._stream
        s.wait_event(self._consumed[j])        # the step that read these buffers has been through them
        return launch_batch(self.dataset, recs, self.tcols, self.nc_theta, self.radius, self._stages[j], s)

    def __iter__(self):
        main = torch.cuda.current_stream(self.dataset.device)
        self._stream.wait_stream(main)
        nb = len(self)
        if not nb:
            return
        nxt = self._launch(0)
        for i in range(nb):
            j = i & 1
            imgs, rows, stage = nxt
            if i + 1 < nb:
                nxt = self._launch(j ^ 1)
            stage.ready.synchronize()          # the side stream only: the compute stream keeps its queue
            nt = int(stage.nt_h.item())
            main.wait_event(stage.ready)
            yield imgs, rows[:nt * self.tcols].view(nt, self.tcols)
            self._consumed[j].record(main)
