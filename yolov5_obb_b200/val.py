"""Validation on the device: val.py:180-276 / 330-333 and utils/metrics.py:15-114.
* match_batch: the per-image metric block of the reference's validation loop (val.py:209-250 and process_batch :69-92),
  executed for a whole batch by ONE kernel (csrc/val_match.cu, SURVEY section 8f rank 3);
* ValStats: the stats list kept on the device and ap_per_class in one call (csrc/val_metrics.cu);
* Validator: the whole loop over a dataloader's batches, returning ValMetrics (results, maps, fitness)."""
from typing import Optional

import torch

from . import _lib
from .dota_eval import _resolve


def match_batch(dets: torch.Tensor, counts: torch.Tensor, targets: torch.Tensor, shapes, iouv: torch.Tensor,
                want_geometry: bool = True):
    """dets [B, max_det, 7] + counts [>= B] int64: the packed pair non_max_suppression_obb(..., return_packed=True / "async")
    returns (rows (cx, cy, l, s, theta, conf, cls) in network-input pixels).
    targets [nt, >= 7]: (image, cls, cx, cy, l, s, theta, ...) as val.py:199 holds them (pixels).
    shapes: per image ((h_raw, w_raw), ((gain_h, gain_w), (pad_x, pad_y))) - the dataloader's `shapes[si]` (val.py:213,233).
    iouv: the IoU thresholds (val.py:165 torch.linspace(0.5, 0.95, 10)).
    Returns (correct [B, max_det, niou] bool, pred_polyn [B, max_det, 8], pred_hbbn [B, max_det, 4]); rows >= counts[b] are
    unspecified for the geometry and False for `correct`.  Everything stays on the device; no synchronisation."""
    _lib.require_cuda(dets, "dets")
    B, max_det, _ = dets.shape
    dev = dets.device
    d = dets.detach().float().contiguous()
    cnt = counts.detach().to(torch.int64).contiguous()
    tg = targets.detach().float()[:, :7].contiguous() if targets.numel() else torch.zeros((0, 7), device=dev)
    sc = torch.tensor([[float(s[1][0][0]), float(s[1][1][0]), float(s[1][1][1]), float(s[0][0]), float(s[0][1])] for s in shapes],
                      dtype=torch.float32).pin_memory().to(dev, non_blocking=True)  # (a pageable copy would drain the stream)
    iv = iouv.detach().float().contiguous().to(dev)
    correct = torch.empty((B, max_det, iv.numel()), dtype=torch.uint8, device=dev)
    polyn = torch.empty((B, max_det, 8), dtype=torch.float32, device=dev) if want_geometry else None
    hbbn = torch.empty((B, max_det, 4), dtype=torch.float32, device=dev) if want_geometry else None
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().y5obb_val_match_f32(d.data_ptr(), cnt.data_ptr(), B, max_det, _lib.ptr(tg) if tg.numel() else None,
                                            tg.shape[0], sc.data_ptr(), iv.data_ptr(), iv.numel(), correct.data_ptr(),
                                            _lib.ptr(polyn), _lib.ptr(hbbn), flag.data_ptr(), _lib.stream_ptr(dev))
    _lib.check(rc, "y5obb_val_match_f32")
    return correct.bool(), polyn, hbbn


# ---------------------------------------------------------------------------------------------------------------------------
# Validation metrics: val.py:209-276 / 330-332 and utils/metrics.py:15-114 (csrc/val_metrics.cu)

GRID = 1000          # ap_per_class's px = np.linspace(0, 1, 1000)
EPS = 1e-16
FITNESS_W = [0.0, 0.0, 0.1, 0.9]  # P, R, mAP@0.5, mAP@0.5:0.95


def fitness(x):
    """utils/metrics.py:15-18: x [n, >= 4] rows (P, R, mAP@.5, mAP@.5:.95, ...) -> [n] weighted sums."""
    return (x[:, :4] * FITNESS_W).sum(1)


class ValMetrics:
    """What val.run returns after the loop, for the classes with labels (np.unique of the target classes):
    `results` (mp, mr, map50, map), `maps` [nc] (per-class mAP@.5:.95, the mean for classes without labels), and per class
    `p`, `r` (at the largest mean F1), `ap50`, `ap` (mAP@.5:.95), `ap_class`; `nt` [nc] labels per class and `seen` images.
    `p_curve` / `r_curve` [n_u, 1000] and `ap_full` [n_u, niou] are ap_per_class's curves and APs.  When no row is a true
    positive at any threshold (val.py:270) every metric is 0 and the per-class arrays are empty."""

    def __init__(self, nc, seen, nt, n_u, ap_class, ap_full, p_curve, r_curve, any_tp):
        import numpy as np
        self.nc, self.seen, self.nt = nc, seen, nt
        self.ap_class = ap_class[:n_u].astype(np.int32)
        self.p_curve, self.r_curve, self.ap_full = p_curve[:n_u], r_curve[:n_u], ap_full[:n_u]
        mp = mr = map50 = map_ = 0.0
        empty = np.zeros(0)
        self.p = self.r = self.f1 = self.tp = self.fp = self.ap50 = self.ap = empty
        if any_tp:
            p, r = self.p_curve, self.r_curve
            n_l = nt[self.ap_class]
            f1 = 2 * p * r / (p + r + EPS)
            i = f1.mean(0).argmax()
            self.p, self.r, self.f1 = p[:, i], r[:, i], f1[:, i]
            self.tp = (self.r * n_l).round()
            self.fp = (self.tp / (self.p + EPS) - self.tp).round()
            self.ap50, self.ap = self.ap_full[:, 0], self.ap_full.mean(1)
            mp, mr, map50, map_ = self.p.mean(), self.r.mean(), self.ap50.mean(), self.ap.mean()
        else:
            self.ap_class = np.zeros(0, np.int32)
        self.results = (mp, mr, map50, map_)
        self.maps = np.zeros(nc) + map_
        for i, c in enumerate(self.ap_class):
            self.maps[c] = self.ap[i]

    def fitness(self):
        """train.py:377 fitness(np.array(results).reshape(1, -1)): [1] = 0.1 mAP@.5 + 0.9 mAP@.5:.95."""
        import numpy as np
        return fitness(np.array(self.results).reshape(1, -1))


class ValStats:
    """The stats list of val.py:209-250 kept on the device: per valid NMS row tp [niou], conf, cls and its (image, row)
    position, and the label count per class nt [nc].  add() is asynchronous (no host read); metrics() computes ap_per_class
    with one synchronisation.  Buffers grow by doubling from the known bound (B * max_det rows per call) with
    device-to-device copies."""

    def __init__(self, nc: int, niou: int = 10, device="cuda"):
        self.nc, self.niou, self.device = int(nc), int(niou), _resolve(device)
        if self.device.type != "cuda":
            raise RuntimeError("ValStats needs a CUDA device; there is no CPU path")
        if self.nc < 1 or self.niou < 1:
            raise RuntimeError("ValStats needs nc >= 1 and niou >= 1")
        dev = self.device
        self.cap, self._bound, self.seen, self._ordered = 0, 0, 0, True
        self._tp = torch.empty((0, self.niou), dtype=torch.uint8, device=dev)
        self._conf = torch.empty(0, dtype=torch.float32, device=dev)
        self._cls = torch.empty(0, dtype=torch.int32, device=dev)
        self._key = torch.empty(0, dtype=torch.int64, device=dev)
        self._n_rows = torch.zeros(1, dtype=torch.int64, device=dev)
        self.nt = torch.zeros(self.nc, dtype=torch.int64, device=dev)
        self._flags = torch.zeros(3, dtype=torch.int32, device=dev)

    def _reserve(self, rows: int) -> None:
        need = self._bound + rows
        if need > self.cap:
            cap = max(self.cap, 1024)
            while cap < need:
                cap *= 2
            grown = []
            for t in (self._tp, self._conf, self._cls, self._key):
                g = torch.empty((cap,) + tuple(t.shape[1:]), dtype=t.dtype, device=self.device)
                g[:self.cap].copy_(t)
                grown.append(g)
            self._tp, self._conf, self._cls, self._key = grown
            self.cap = cap
        self._bound = need

    def add(self, dets: torch.Tensor, counts: torch.Tensor, correct: torch.Tensor, targets: torch.Tensor,
            nms_cap: Optional[int] = None, image_base: Optional[int] = None) -> torch.Tensor:
        """dets [B, max_det, 7] fp32 and counts int64 (the packed NMS output), correct [B, max_det, niou] bool / uint8
        (match_batch), targets [nt, >= 2] fp32 (image, cls, ...).  With nms_cap (non_max_suppression_obb's async form:
        counts has B + 1 entries) a batch whose candidates overflowed the NMS capacity is not appended at all.  image_base:
        the first image index of a batch added again (its rows keep their (image, row) positions); by default the batch's
        images follow the ones seen so far.  Returns the device int32 [1] skip flag (1 = not appended)."""
        for t, name in ((dets, "dets"), (counts, "counts"), (correct, "correct"), (targets, "targets")):
            _lib.require_cuda(t, name)
            if t.device != self.device:
                raise RuntimeError(f"{name} is on {t.device}, the stats on {self.device}")
        if dets.dtype != torch.float32 or dets.dim() != 3 or dets.shape[2] != 7:
            raise RuntimeError(f"dets must be fp32 [B, max_det, 7], got {dets.dtype} {tuple(dets.shape)}")
        B, max_det = dets.shape[0], dets.shape[1]
        if counts.dtype != torch.int64 or counts.dim() != 1 or counts.numel() < B + (nms_cap is not None):
            raise RuntimeError(f"counts must be int64 [{B}{' + 1' if nms_cap is not None else ''}], got {counts.dtype} "
                               f"{tuple(counts.shape)}")
        if correct.dtype not in (torch.bool, torch.uint8) or tuple(correct.shape) != (B, max_det, self.niou):
            raise RuntimeError(f"correct must be bool / uint8 [{B}, {max_det}, {self.niou}], got {correct.dtype} "
                               f"{tuple(correct.shape)}")
        if targets.dtype != torch.float32 or targets.dim() != 2 or (targets.shape[0] and targets.shape[1] < 2):
            raise RuntimeError(f"targets must be fp32 [nt, >= 2], got {targets.dtype} {tuple(targets.shape)}")
        if image_base is None:
            image_base = self.seen
            self.seen += B
        else:
            self._ordered = False
        self._reserve(B * max_det)
        d, c, cor = dets.contiguous(), counts.contiguous(), correct.contiguous().view(torch.uint8)
        tg = targets.contiguous()
        skip = torch.empty(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_val_stats_append(
                d.data_ptr(), c.data_ptr(), B, max_det, -1 if nms_cap is None else int(nms_cap), cor.data_ptr(), self.niou,
                tg.data_ptr() if tg.numel() else None, tg.shape[0] if tg.numel() else 0, tg.shape[1] if tg.numel() else 2,
                int(image_base), self._tp.data_ptr(), self._conf.data_ptr(), self._cls.data_ptr(), self._key.data_ptr(),
                self.cap, self._n_rows.data_ptr(), self.nt.data_ptr(), self.nc, self._flags.data_ptr(), skip.data_ptr(),
                _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_val_stats_append")
        return skip

    def rows(self):
        """(tp [n, niou] uint8, conf, cls, key) of the appended rows, in append order (reads the row count)."""
        n = int(self._n_rows.item())
        return self._tp[:n], self._conf[:n], self._cls[:n], self._key[:n]

    def metrics(self) -> ValMetrics:
        """ap_per_class (csrc/val_metrics.cu y5obb_ap_per_class_f64) over everything added, then one read to the host and
        the small tail of val.py in numpy.  Raises RuntimeError when a class was outside [0, nc)."""
        import numpy as np
        nc, niou, dev = self.nc, self.niou, self.device
        ap = torch.empty((nc, niou), dtype=torch.float64, device=dev)
        p = torch.empty((nc, GRID), dtype=torch.float64, device=dev)
        r = torch.empty((nc, GRID), dtype=torch.float64, device=dev)
        ap_class = torch.empty(nc, dtype=torch.int32, device=dev)
        n_u = torch.empty(1, dtype=torch.int32, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            need = L.y5obb_ap_per_class_workspace_bytes(self.cap, niou, nc)
            ws = _lib.workspace(need, dev, f"val_metrics:{_lib.stream_ptr(dev)}")
            _lib.check(L.y5obb_ap_per_class_f64(
                _lib.ptr(self._tp), _lib.ptr(self._conf), _lib.ptr(self._cls), _lib.ptr(self._key), self._n_rows.data_ptr(),
                self.cap, int(self._ordered), self.nt.data_ptr(), nc, niou, ap.data_ptr(), p.data_ptr(), r.data_ptr(),
                ap_class.data_ptr(), n_u.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)),
                "y5obb_ap_per_class_f64")
            h = torch.cat([self._flags[:2].double(), n_u.double(), ap_class.double(), self.nt.double(), ap.flatten(),
                           p.flatten(), r.flatten()]).cpu().numpy()   # the one synchronisation
        if int(h[0]) & 1:
            raise RuntimeError("ValStats: a detection or label class is outside [0, nc)")
        if int(h[0]) & 2:
            raise RuntimeError("ValStats: rows past the buffer capacity")
        o = 3
        ac = h[o:o + nc].astype(np.int64)
        nt = h[o + nc:o + 2 * nc].astype(np.int64)
        o += 2 * nc
        apf = h[o:o + nc * niou].reshape(nc, niou).copy()
        o += nc * niou
        pc = h[o:o + nc * GRID].reshape(nc, GRID).copy()
        rc = h[o + nc * GRID:].reshape(nc, GRID).copy()
        return ValMetrics(nc, self.seen, nt, int(h[2]), ac, apf, pc, rc, bool(h[1]))


def _upload(t: torch.Tensor, device) -> torch.Tensor:
    if t.is_cuda:
        return t
    return (t if t.is_pinned() else t.pin_memory()).to(device, non_blocking=True)


class Validator:
    """val.py:180-250 for a model in eval mode, then ValStats.metrics(): `Validator(model)(batches)` -> ValMetrics, where
    batches yields the dataloader's (im, targets, paths, shapes): im uint8 [B, 3, H, W], targets fp32 [nt, >= 7] (image,
    cls, cx, cy, l, s, theta, ...) in network-input pixels, shapes per image ((h_raw, w_raw), ((gain, gain), (pad_x, pad_y))).
    Per batch: upload, detect_records, non_max_suppression_obb(return_packed="async"), match_batch, ValStats.add - no host
    read.  A batch whose NMS candidates overflowed the optimistic capacity is not appended; its skip flag is read one batch
    late, while the next batch computes, and the batch is then re-run with the blocking NMS from its device copy.
    compute_loss (a loss.ComputeLoss, train.py:364-373): the validation loss of val.py:198-199 is added per batch from the
    plan's Detect inputs (ComputeLoss.head_items) into a device fp32 sum, and `results` becomes val.py:333's
    (mp, mr, map50, map, box, obj, cls, theta) with the loss sum divided by the number of batches.
    Raw form: `im` may be the list of the batch's decoded source images (uint8 [h0, w0, 3] BGR arrays of any sizes) instead
    of the letterboxed tensor.  `shapes` then says where each one lands (letterbox.place_rect(...).shapes, the rect loader's
    entry); csrc/letterbox.cu resamples them as load_image_label + letterbox do and writes the plan's stem input, and
    everything after the forward is the same.  targets stay in network-input pixels (Placement.map_labels).
    `model` may be an ensemble.Ensemble (val.py --weights a.pt b.pt); it has no validation loss."""

    def __init__(self, model, conf_thres: float = 0.01, iou_thres: float = 0.4, max_det: int = 1500, iouv=None,
                 augment: bool = False, compute_loss=None):
        from .ensemble import Ensemble
        if compute_loss is not None and isinstance(model, Ensemble):
            # val.py run on an ensemble has no loss: train.py validates the single EMA model (val.py:198, compute_loss)
            raise RuntimeError("the validation loss is defined for a single model, not an ensemble")
        self.model = model
        self.augment = bool(augment)   # val.py --augment: test-time augmentation (Model.detect_records(augment=True))
        self.device = _resolve(next(model.parameters()).device)
        if self.device.type != "cuda":
            raise RuntimeError("Validator needs the model on a CUDA device; there is no CPU path")
        if compute_loss is not None and not hasattr(compute_loss, "head_items"):
            raise RuntimeError("compute_loss must be a yolov5_obb_b200.loss.ComputeLoss (the loss is computed from the eval "
                               "plan's Detect inputs)")
        if compute_loss is not None and self.augment:
            # the reference has no training outputs under augmentation either (train_out = None, val.py:199)
            raise RuntimeError("the validation loss is not defined with test-time augmentation")
        self.compute_loss = compute_loss
        self.nms = dict(conf_thres=conf_thres, iou_thres=iou_thres, multi_label=True, max_det=max_det)
        iouv = torch.linspace(0.5, 0.95, 10) if iouv is None else iouv
        self.iouv = iouv.detach().float().to(self.device)
        self.reruns = 0
        self._raw_host, self._raw_ev, self._raw_n = [None, None], [None, None], 0   # pinned buffers of the raw form

    def _upload_raw(self, images, shapes):
        """The batch's source images, packed and uploaded with one copy -> (device buffer, letterbox.PackedBatch)."""
        from . import letterbox as lb
        if self.augment:
            raise RuntimeError("test-time augmentation reads the letterboxed tensor: pass `im` as a tensor with augment=True")
        if len(images) != len(shapes):
            raise RuntimeError(f"{len(images)} images but {len(shapes)} shapes entries")
        placed = [lb.place_from_shapes(s) for s in shapes]
        hw = {p[1] for p in placed}
        if len(hw) != 1:
            raise RuntimeError(f"the shapes entries of one batch describe different letterboxed sizes: {sorted(hw)}")
        (Hp, Wp), = hw
        k = self._raw_n % 2
        self._raw_n += 1
        if self._raw_ev[k] is not None:
            self._raw_ev[k].synchronize()   # the upload that last read this pinned buffer
        batch = lb.pack_batch([lb.as_image(im) for im in images], [p[0] for p in placed], Hp, Wp, self._raw_host[k])
        self._raw_host[k] = batch.host
        buf = batch.host[:batch.nbytes].to(self.device, non_blocking=True)
        self._raw_ev[k] = torch.cuda.Event()
        self._raw_ev[k].record()
        return buf, batch

    def _records(self, x):
        """detect_records for either form of a batch -> (DetectRecords, the plan's input shape)."""
        if isinstance(x, torch.Tensor):
            return self.model.detect_records(x, augment=self.augment), tuple(x.shape)
        from . import letterbox as lb
        buf, batch = x
        return lb.letterboxed_records(self.model, buf, batch, self.device)[0], (batch.B, 3, batch.Hp, batch.Wp)

    def __call__(self, batches) -> ValMetrics:
        nc = self.model.nc if hasattr(self.model, "nc") else self.model.model[-1].nc   # (an Ensemble has `nc`)
        stats = ValStats(nc, self.iouv.numel(), self.device)
        pending = None
        self._loss, n_batches = torch.zeros(4, dtype=torch.float32, device=self.device), 0
        with torch.cuda.device(self.device):
            for im, targets, _paths, shapes in batches:
                cur = self._submit(stats, im, targets, shapes)
                n_batches += 1
                if pending is not None:
                    self._settle(stats, pending)
                pending = cur
            if pending is not None:
                self._settle(stats, pending)
            m = stats.metrics()
        if self.compute_loss is not None:
            m.results = m.results + tuple((self._loss.cpu() / n_batches).tolist())   # val.py:333
        return m

    def _submit(self, stats, im, targets, shapes):
        from .general import non_max_suppression_obb
        x = self._upload_raw(im, shapes) if isinstance(im, (list, tuple)) else _upload(im, self.device)
        t = _upload(targets.float(), self.device)
        base = stats.seen
        recs, shape = self._records(x)
        if self.compute_loss is not None:   # val.py:198-199; the overflow re-run in _settle does not add it again
            self._loss += self.compute_loss.head_items(self.model.records_plan(shape, self.device), t)[1]
        dets, counts, cap = non_max_suppression_obb(recs, return_packed="async", **self.nms)
        correct, _, _ = match_batch(dets, counts, t, shapes, self.iouv, want_geometry=False)
        skip = stats.add(dets, counts, correct, t, nms_cap=cap)
        host = torch.empty(1, dtype=torch.int32).pin_memory()
        host.copy_(skip, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return host, ev, x, t, shapes, base

    def _settle(self, stats, pending):
        from .general import non_max_suppression_obb
        host, ev, x, t, shapes, base = pending
        ev.synchronize()
        if int(host[0]) == 0:
            return
        self.reruns += 1
        dets, rows = non_max_suppression_obb(self._records(x)[0], return_packed=True, **self.nms)
        counts = torch.tensor(rows, dtype=torch.int64).to(self.device)
        correct, _, _ = match_batch(dets, counts, t, shapes, self.iouv, want_geometry=False)
        stats.add(dets, counts, correct, t, image_base=base)
