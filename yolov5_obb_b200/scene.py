"""Whole-scene DOTA inference on the device: the reference's documented route for scenes larger than one tile
(README.md:24-26, docs/GetStart.md:117-130) in one call.

The reference cuts the scene into tiles with DOTA_devkit/ImgSplit_multi_process.py (PNG files), detects every tile with
`val.py --task test --save-json`, rewrites the JSON per class (tools/TestJson2VocClassTxt.py) and merges the tiles with
DOTA_devkit/ResultMerge_multi_process.py (polygon NMS per scene and class, 16 CPU processes).  Here the decoded scene stays
on the device: csrc/scene.cu writes the stem input of each batch of tiles straight into the records plan, the batched
post-process runs as usual, and one merge pass reproduces the rounding, the shift into scene coordinates and the per-class
polygon NMS of the reference chain bit for bit (DESIGN.md section 4 and section 7 for tied scores)."""
import math
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .general import DetectRecords, non_max_suppression_obb


def split_origins(height: int, width: int, subsize: int = 1024, gap: int = 200) -> List[Tuple[int, int]]:
    """Tile origins (left, up) in the order of ImgSplit_multi_process.py SplitSingle at rate 1 (:251-273): columns outer,
    rows inner, a slide of subsize - gap, the last column / row clamped to max(size - subsize, 0)."""
    if gap >= subsize or gap < 0:
        raise RuntimeError(f"gap ({gap}) must be in [0, subsize) (subsize {subsize})")
    slide = subsize - gap
    out = []
    left = 0
    while left < width:
        if left + subsize >= width:
            left = max(width - subsize, 0)
        up = 0
        while up < height:
            if up + subsize >= height:
                up = max(height - subsize, 0)
            out.append((left, up))
            if up + subsize >= height:
                break
            up += slide
        if left + subsize >= width:
            break
        left += slide
    return out


def tile_geometry(subsize: int = 1024, pad: float = 0.5, stride: int = 32) -> Tuple[int, int, float]:
    """(size, border, pad_xy): the inference size of a tile as val.py's rect batching makes it with the model's largest
    stride, ceil(subsize / stride + pad) * stride (utils/datasets.py:492; 1056 for a P5 model, 1088 for a P6 model at subsize
    1024 and pad 0.5), the letterbox border on the top / left, int(round(d - 0.1)) with d = (size - subsize) / 2, and d
    itself, which scale_polys subtracts (utils/augmentations.py:92-128 with auto=False, scaleup=False)."""
    if pad < 0:
        raise RuntimeError(f"pad must be >= 0, got {pad}")
    if stride < 1:
        raise RuntimeError(f"stride must be >= 1, got {stride}")
    size = int(math.ceil(subsize / stride + pad)) * stride
    d = (size - subsize) / 2
    return size, int(round(d - 0.1)), d


class SceneDetections:
    """Merged detections of one scene: `rows` [K, 10] fp64 on the device, (class, score, x1 y1 x2 y2 x3 y3 x4 y4) in scene
    pixels, classes ascending and each class in keep order.  Score and coordinates are the values the reference's merge holds
    (round(conf, 5), round(x, 1) + tile origin); write_task1 applies its final rounding."""

    def __init__(self, data: torch.Tensor, n: torch.Tensor):
        self._data, self._n, self._rows = data, n, None

    @property
    def rows(self) -> torch.Tensor:
        if self._rows is None:  # K is read on first use
            self._rows = self._data[:int(self._n.item())]
        return self._rows

    def per_class(self) -> Dict[int, torch.Tensor]:
        """{class: [k, 10] rows} for the classes that have detections."""
        rows = self.rows
        cls, cnt = torch.unique_consecutive(rows[:, 0], return_counts=True)
        return {int(c): r for c, r in zip(cls.tolist(), torch.split(rows, cnt.tolist()))}

    def write_task1(self, dstdir, scene_name: str, names: Sequence[str]) -> None:
        """Appends this scene's lines to dstdir/Task1_<name>.txt in the text format of ResultMerge_multi_process.py mergesingle
        (:221-236): `scene score x1 y1 ... y4` with str(round(score, 2)) and str(round(x, 1))."""
        os.makedirs(dstdir, exist_ok=True)
        by_class: Dict[int, List[str]] = {}
        for row in self.rows.cpu().tolist():
            line = scene_name + " " + str(round(row[1], 2)) + " " + " ".join(map(str, [round(x, 1) for x in row[2:]]))
            by_class.setdefault(int(row[0]), []).append(line + "\n")
        for c, lines in by_class.items():
            with open(os.path.join(dstdir, f"Task1_{names[c]}.txt"), "a") as f:
                f.writelines(lines)


def merge_tiles(rows: torch.Tensor, counts: torch.Tensor, origins: torch.Tensor, nc: int, pad: float = 16.0,
                thresh: float = 0.2) -> SceneDetections:
    """Tile-merge of packed per-tile detections (csrc/scene.cu y5obb_scene_merge_f64): rows [T, max_det, 7] fp32
    (cx, cy, l, s, theta, conf, cls) with counts [T] int64 valid rows each, as non_max_suppression_obb(return_packed=...)
    leaves them, and origins [T, 2] int32 (left, up), all on one CUDA device; pad is the letterbox offset scale_polys removes.
    Synchronises the stream once (the per-class candidate counts size the suppression masks)."""
    for t, name in ((rows, "rows"), (counts, "counts"), (origins, "origins")):
        _lib.require_cuda(t, name)
    T, max_det = rows.shape[0], rows.shape[1]
    if rows.dtype != torch.float32 or rows.dim() != 3 or rows.shape[2] != 7 or counts.dtype != torch.int64 or \
            origins.dtype != torch.int32 or tuple(origins.shape) != (T, 2) or counts.shape[0] < T:
        raise RuntimeError("merge_tiles wants rows fp32 [T, max_det, 7], counts int64 [T], origins int32 [T, 2]")
    rows, counts, origins = rows.contiguous(), counts.contiguous(), origins.contiguous()
    dev = rows.device
    L = _lib.lib()
    out10 = torch.empty((T * max_det, 10), dtype=torch.float64, device=dev)
    n_out = torch.empty(1, dtype=torch.int64, device=dev)
    cands = np.zeros(nc, np.int64)
    need = L.y5obb_scene_merge_workspace_bytes(T, max_det, nc, None)
    with torch.cuda.device(dev):
        while True:
            ws = _lib.workspace(need, dev, f"scene_merge:{_lib.stream_ptr(dev)}")
            rc = L.y5obb_scene_merge_f64(rows.data_ptr(), counts.data_ptr(), origins.data_ptr(), T, max_det, nc, float(pad), 1.0,
                                         float(thresh), out10.data_ptr(), n_out.data_ptr(), cands.ctypes.data, ws.data_ptr(),
                                         ws.numel(), _lib.stream_ptr(dev))
            if rc == 1 and cands.max() > _lib.SCENE_MAX_CLASS_CANDIDATES:
                c = int(cands.argmax())
                raise RuntimeError(f"class {c} has {int(cands[c])} merge candidates in this scene: the dense polygon-NMS mask "
                                   f"is bounded at {_lib.SCENE_MAX_CLASS_CANDIDATES} candidates per class "
                                   "(Y5OBB_SCENE_MAX_CLASS_CANDIDATES)")
            if rc != 2:
                break
            need = L.y5obb_scene_merge_workspace_bytes(T, max_det, nc, cands.ctypes.data)
    _lib.check(rc, "y5obb_scene_merge_f64")
    return SceneDetections(out10, n_out)


class SceneDetector:
    """Scene (uint8 [H, W, 3] BGR on a CUDA device, as cv2.imread decodes it) -> SceneDetections, as the reference's
    ImgSplit (rate 1) -> val.py --conf conf_thres --iou iou_thres --save-json -> TestJson2VocClassTxt -> ResultMerge chain
    computes them.  Tiles run in batches of batch_size through one records plan; the last batch runs the full plan and the
    detections of its padding tiles are ignored.  pad=0.5 is val.py's rect-batching pad (1056^2 tiles for subsize 1024,
    1088^2 for a stride-64 P6 model: the size is rounded to the model's largest stride), pad=0.0 the unpadded tile of detect.py /
    --task speed.  The model is one of the two families the engine plans: P5 (strides 8, 16, 32) or P6 (8, 16, 32, 64), or an
    ensemble.Ensemble of them, whose stride is its largest member's (1088^2 tiles as soon as one member is a P6 model)."""

    def __init__(self, model, batch_size: int = 16, subsize: int = 1024, gap: int = 200, conf_thres: float = 0.01,
                 iou_thres: float = 0.4, max_det: int = 1500, merge_thresh: float = 0.2, pad: float = 0.5):
        if gap >= subsize or gap < 0:
            raise RuntimeError(f"gap ({gap}) must be in [0, subsize) (subsize {subsize})")
        if batch_size < 1 or max_det < 1:
            raise RuntimeError("batch_size and max_det must be >= 1")
        strides = [float(v) for v in model.stride]
        if strides not in ([8.0, 16.0, 32.0], [8.0, 16.0, 32.0, 64.0]):
            raise RuntimeError(f"the model's Detect strides {strides} are neither the P5 layout (8, 16, 32) of yolov5*.yaml nor "
                               "the P6 layout (8, 16, 32, 64) of models/hub/yolov5*6.yaml")
        self.size, self.border, self.pad_xy = tile_geometry(subsize, pad, int(strides[-1]))
        self.model, self.B, self.subsize, self.gap = model, int(batch_size), int(subsize), int(gap)
        self.conf_thres, self.iou_thres, self.max_det, self.merge_thresh = conf_thres, iou_thres, int(max_det), merge_thresh
        self._status_host = None

    def det(self, scene: torch.Tensor) -> SceneDetections:
        if not scene.is_cuda:
            raise RuntimeError("the scene must be a CUDA tensor: there is no CPU path")
        if scene.dtype != torch.uint8 or scene.dim() != 3 or scene.shape[2] != 3:
            raise RuntimeError(f"the scene must be uint8 [H, W, 3] (BGR), got {scene.dtype} {tuple(scene.shape)}")
        scene = scene.contiguous()
        dev = scene.device
        H, W = scene.shape[0], scene.shape[1]
        origins = split_origins(H, W, self.subsize, self.gap)
        T, B = len(origins), self.B
        nb = (T + B - 1) // B
        org = torch.tensor(origins, dtype=torch.int32).to(dev)
        rows = torch.empty((T, self.max_det, 7), dtype=torch.float32, device=dev)
        counts = torch.empty(T, dtype=torch.int64, device=dev)
        status = torch.empty((nb, 2), dtype=torch.int64, device=dev)   # per batch: (candidates found, capacity)
        with torch.cuda.device(dev):
            for i in range(nb):
                self._run_batch(scene, org, i, rows, counts, status[i])
            if self._status_host is None or self._status_host.shape[0] < nb:
                self._status_host = torch.empty((nb, 2), dtype=torch.int64).pin_memory()
            st_host = self._status_host[:nb]
            st_host.copy_(status, non_blocking=True)   # complete once the merge has synchronised the stream
            out = merge_tiles(rows, counts, org, self.nc, self.pad_xy, self.merge_thresh)
            bad = [i for i, (found, cap) in enumerate(st_host.tolist()) if found < 0 or found > cap]
            if bad:   # rare: a batch had more NMS candidates than the optimistic capacity; re-run it with the blocking form
                for i in bad:
                    self._run_batch(scene, org, i, rows, counts, None)
                out = merge_tiles(rows, counts, org, self.nc, self.pad_xy, self.merge_thresh)
        return out

    def _run_batch(self, scene, org, i, rows, counts, status):
        B, T = self.B, counts.shape[0]
        t0 = i * B
        n = min(B, T - t0)
        dev = scene.device
        eng = self.model.records_plan((B, 3, self.size, self.size), dev)
        name = "y5obb_scene_tiles_s2d_u8" + ("_f16" if eng.half else "")
        _lib.check(getattr(_lib.lib(), name)(scene.data_ptr(), scene.shape[0], scene.shape[1], org[t0].data_ptr(), n,
                                             self.subsize, self.size, self.border, eng.x_s2d.data_ptr(), 1,
                                             _lib.stream_ptr(dev)), name)
        rec = DetectRecords(eng.forward_s2d(), eng.nc, eng.half)
        self.nc = eng.nc
        kw = dict(multi_label=True, max_det=self.max_det)
        if status is None:
            out, c = non_max_suppression_obb(rec, self.conf_thres, self.iou_thres, return_packed=True, **kw)
            rows[t0:t0 + n].copy_(out[:n])
            counts[t0:t0 + n].copy_(torch.tensor(c[:n], dtype=torch.int64))
            return
        out, c, cap = non_max_suppression_obb(rec, self.conf_thres, self.iou_thres, return_packed="async", **kw)
        rows[t0:t0 + n].copy_(out[:n])   # (the post-process outputs are graph-owned: copied before the next batch)
        counts[t0:t0 + n].copy_(c[:n])
        status[0].copy_(c[B])
        status[1].fill_(cap)
