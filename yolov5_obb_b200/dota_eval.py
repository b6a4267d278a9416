"""DOTA Task1 evaluation on the device: the OBB mAP the reference reports (README / docs/GetStart.md step 4,
DOTA_devkit/dota_evaluation_task1.py) in one call.

The reference reads the Task1_<class>.txt files and the labelTxt ground truth back from disk, then walks every detection of
every class in Python with one polyiou call per candidate pair.  Here csrc/dota_eval.cu sorts, matches, builds the precision /
recall curves and computes the VOC AP of every class in one asynchronous pass that reproduces voc_eval and voc_ap bit for bit
(DESIGN.md section 4; tied scores keep input order, section 7).  Two routes feed it:
  * files: load_gt + load_task1 parse labelTxt and Task1 files as the reference does;
  * memory: Task1Detections.add takes SceneDetections straight from SceneDetector.det and applies write_task1's rounding on
    the device, so evaluating it equals evaluating the files write_task1 would have written."""
import math
import os
from typing import List, Optional, Sequence

import torch

from . import _lib


def _image_index(imagenames: Sequence[str]) -> dict:
    idx = {}
    for i, name in enumerate(imagenames):
        if name in idx:
            raise RuntimeError(f"image name {name!r} appears twice in imagenames")
        idx[name] = i
    return idx


def _resolve(device) -> torch.device:
    """torch.device with the index filled in: a bare "cuda" is the current CUDA device, so that it compares equal to the
    device of the tensors made there."""
    d = torch.device(device)
    if d.type == "cuda" and d.index is None:
        d = torch.device("cuda", torch.cuda.current_device())
    return d


class GroundTruth:
    """Ground-truth objects of an image set: `img` int32 [n] (index into imagenames) and `rows` fp64 [n, 10] (class,
    difficult, x1 y1 ... x4 y4), images in imagenames order and each file's objects in line order."""

    def __init__(self, img: torch.Tensor, rows: torch.Tensor, imagenames: Sequence[str], nc: int):
        self.img, self.rows, self.imagenames, self.nc = img, rows, list(imagenames), int(nc)


def load_gt(annopath_fmt: str, imagenames: Sequence[str], classnames: Sequence[str], device="cuda") -> GroundTruth:
    """labelTxt files annopath_fmt.format(image) parsed as parse_gt (dota_evaluation_task1.py:22-53) does: lines of fewer
    than 9 space-separated tokens (the imagesource: / gsd: headers) are skipped, coordinates are Python floats, difficult is
    int(token 9) (0 without it; any non-zero value is difficult).  Objects whose name is not in classnames are ignored.  An
    object line of a listed class with more than 10 tokens raises RuntimeError: parse_gt leaves its `difficult` unset and
    voc_eval then stops with a KeyError."""
    _image_index(imagenames)
    cls_idx = {n: c for c, n in enumerate(classnames)}
    img: List[int] = []
    rows: List[List[float]] = []
    for i, name in enumerate(imagenames):
        with open(annopath_fmt.format(name), "r") as f:
            for line in f:
                tok = line.strip().split(" ")
                if len(tok) < 9 or tok[8] not in cls_idx:
                    continue
                if len(tok) > 10:
                    raise RuntimeError(f"{annopath_fmt.format(name)}: an object line has 9 or 10 fields (x1 y1 ... x4 y4 "
                                       f"class [difficult]), got {line!r}")
                difficult = int(tok[9]) if len(tok) > 9 else 0
                rows.append([float(cls_idx[tok[8]]), float(difficult)] + [float(t) for t in tok[:8]])
                img.append(i)
    return GroundTruth(torch.tensor(img, dtype=torch.int32).to(device),
                       torch.tensor(rows, dtype=torch.float64).reshape(-1, 10).to(device), imagenames, len(classnames))


class Task1Detections:
    """Detections of an image set in Task1 form: `img` int32 [n] and `rows` fp64 [n, 10] (class, score, x1 y1 ... x4 y4)
    in input order, which decides between tied scores (lower first).  A class is present (it counts in the mAP) when its
    Task1 file exists (load_task1) or, for detections added from scenes, when it has at least one detection, which is when
    write_task1 creates its file."""

    def __init__(self, imagenames: Sequence[str], nc: int, device="cuda"):
        self.imagenames, self.nc, self.device = list(imagenames), int(nc), _resolve(device)
        self._index = _image_index(self.imagenames)
        self._img: List[torch.Tensor] = []
        self._rows: List[torch.Tensor] = []
        self._cat = None
        self.present_host: Optional[List[bool]] = None   # set by load_task1: the classes whose file exists

    def add(self, image_index: int, scene) -> "Task1Detections":
        """Appends one scene's merged detections (SceneDetections, rows [K, 10] fp64 on the device) as the detections of
        imagenames[image_index], rounded as write_task1 writes them: round(score, 2), round(x, 1).  Reads K once."""
        if not 0 <= int(image_index) < len(self.imagenames):
            raise RuntimeError(f"image index {image_index} is outside [0, {len(self.imagenames)})")
        rows = scene.rows
        _lib.require_cuda(rows, "scene rows")
        if rows.dtype != torch.float64 or rows.dim() != 2 or rows.shape[1] != 10 or rows.device != self.device:
            raise RuntimeError(f"scene rows must be fp64 [K, 10] on {self.device}, got {rows.dtype} {tuple(rows.shape)} "
                               f"on {rows.device}")
        rows = rows.contiguous()
        out = torch.empty_like(rows)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().y5obb_task1_round_f64(rows.data_ptr(), rows.shape[0], out.data_ptr(),
                                                        _lib.stream_ptr(self.device)), "y5obb_task1_round_f64")
        self._rows.append(out)
        self._img.append(torch.full((rows.shape[0],), int(image_index), dtype=torch.int32, device=self.device))
        self._cat = None
        return self

    def add_rows(self, img: torch.Tensor, rows: torch.Tensor) -> "Task1Detections":
        """Appends detections already in Task1 form: img int32 [n] and rows fp64 [n, 10] (class, score, 8 coordinates), used
        as they are (no rounding).  evaluate_task1 checks them."""
        self._img.append(img)
        self._rows.append(rows)
        self._cat = None
        return self

    def _tensors(self):
        if self._cat is None:
            if self._rows:
                self._cat = (torch.cat(self._img), torch.cat(self._rows))
            else:
                self._cat = (torch.zeros(0, dtype=torch.int32, device=self.device),
                             torch.zeros((0, 10), dtype=torch.float64, device=self.device))
        return self._cat

    @property
    def img(self) -> torch.Tensor:
        return self._tensors()[0]

    @property
    def rows(self) -> torch.Tensor:
        return self._tensors()[1]


def load_task1(detpath_fmt: str, imagenames: Sequence[str], classnames: Sequence[str], device="cuda") -> Task1Detections:
    """Task1 files detpath_fmt.format(class) (`image score x1 y1 ... x4 y4` per line) as voc_eval reads them
    (dota_evaluation_task1.py:145-154), classes in classnames order and lines in file order.  A missing file marks its class
    absent (main() skips it); an image id outside imagenames raises RuntimeError (a KeyError in the reference)."""
    dets = Task1Detections(imagenames, len(classnames), device)
    present = [False] * len(classnames)
    img: List[int] = []
    rows: List[List[float]] = []
    for c, name in enumerate(classnames):
        path = detpath_fmt.format(name)
        if not os.path.exists(path):
            continue
        present[c] = True
        with open(path, "r") as f:
            lines = f.readlines()
        for line in lines:
            tok = line.strip().split(" ")
            if tok[0] not in dets._index:
                raise RuntimeError(f"{path}: image id {tok[0]!r} is not in imagenames")
            if len(tok) != 10:
                raise RuntimeError(f"{path}: a Task1 line has 10 fields (image score x1 y1 ... x4 y4), got {line!r}")
            img.append(dets._index[tok[0]])
            rows.append([float(c), float(tok[1])] + [float(z) for z in tok[2:]])
    dets._img = [torch.tensor(img, dtype=torch.int32).to(device)]
    dets._rows = [torch.tensor(rows, dtype=torch.float64).reshape(-1, 10).to(device)]
    dets.present_host = present
    return dets


class Task1Eval:
    """Result of evaluate_task1.  On the device, without a synchronisation: `ap` fp64 [nc], `npos` int64 [nc] (non-difficult
    GTs), `present` bool [nc], `class_off` int64 [nc + 1].  `map`, `rec(c)`, `prec(c)` and `check()` read the results to
    the host once (the one synchronisation) and raise RuntimeError if a row's class or image was out of range."""

    def __init__(self, ap, npos, present, class_off, rec, prec, status):
        self.ap, self.npos, self.present, self.class_off = ap, npos, present, class_off
        self._rec, self._prec, self._status, self._host = rec, prec, status, None

    def check(self):
        if self._host is None:
            nc = self.ap.shape[0]
            h = torch.cat([self._status.double(), self.ap, self.present.double(), self.class_off.double()]).cpu()
            if int(h[0]) != 0:
                raise RuntimeError("evaluate_task1: a detection or ground-truth row has a class outside [0, nc) or an image "
                                   "outside imagenames")
            self._host = (h[1:1 + nc].tolist(), [bool(x) for x in h[1 + nc:1 + 2 * nc].tolist()],
                          [int(x) for x in h[1 + 2 * nc:].tolist()])
        return self._host

    @property
    def map(self) -> float:
        """main() (dota_evaluation_task1.py:305-343): the sum of the present classes' APs in class order over their number
        (nan when no class is present)."""
        ap, present, _ = self.check()
        m, n = 0.0, 0
        for a, p in zip(ap, present):
            if p:
                m = m + a
                n += 1
        return m / n if n else math.nan

    def rec(self, c: int) -> torch.Tensor:
        off = self.check()[2]
        return self._rec[off[c]:off[c + 1]]

    def prec(self, c: int) -> torch.Tensor:
        off = self.check()[2]
        return self._prec[off[c]:off[c + 1]]


def evaluate_task1(dets: Task1Detections, gt: GroundTruth, ovthresh: float = 0.5, use_07_metric: bool = True) -> Task1Eval:
    """voc_eval + voc_ap of every class (csrc/dota_eval.cu y5obb_dota_eval_f64), asynchronous on the current stream.
    use_07_metric=True is the VOC07 11-point AP that main() uses."""
    det_img, det_rows = dets.img, dets.rows
    for t, name in ((det_img, "detection images"), (det_rows, "detection rows"), (gt.img, "GT images"), (gt.rows, "GT rows")):
        _lib.require_cuda(t, name)
    dev = det_rows.device
    if det_rows.dtype != torch.float64 or det_rows.dim() != 2 or det_rows.shape[1] != 10 or det_img.dtype != torch.int32 or \
            tuple(det_img.shape) != (det_rows.shape[0],):
        raise RuntimeError("detections must be rows fp64 [n, 10] and img int32 [n]")
    if gt.rows.dtype != torch.float64 or gt.rows.dim() != 2 or gt.rows.shape[1] != 10 or gt.img.dtype != torch.int32 or \
            tuple(gt.img.shape) != (gt.rows.shape[0],):
        raise RuntimeError("ground truth must be rows fp64 [m, 10] and img int32 [m]")
    if any(t.device != dev for t in (det_img, gt.img, gt.rows)):
        raise RuntimeError("detections and ground truth must be on one device")
    if dets.nc != gt.nc or len(dets.imagenames) != len(gt.imagenames):
        raise RuntimeError(f"detections ({dets.nc} classes, {len(dets.imagenames)} images) and ground truth ({gt.nc} classes, "
                           f"{len(gt.imagenames)} images) describe different sets")
    nc, n_images = dets.nc, len(dets.imagenames)
    det_img, det_rows, gt_img, gt_rows = det_img.contiguous(), det_rows.contiguous(), gt.img.contiguous(), gt.rows.contiguous()
    n_det, n_gt = det_rows.shape[0], gt_rows.shape[0]
    class_off = torch.empty(nc + 1, dtype=torch.int64, device=dev)
    rec = torch.empty(n_det, dtype=torch.float64, device=dev)
    prec = torch.empty(n_det, dtype=torch.float64, device=dev)
    ap = torch.empty(nc, dtype=torch.float64, device=dev)
    npos = torch.empty(nc, dtype=torch.int64, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        need = L.y5obb_dota_eval_workspace_bytes(n_det, n_gt, n_images, nc)
        ws = _lib.workspace(need, dev, f"dota_eval:{_lib.stream_ptr(dev)}")
        _lib.check(L.y5obb_dota_eval_f64(det_img.data_ptr(), det_rows.data_ptr(), n_det, gt_img.data_ptr(), gt_rows.data_ptr(),
                                         n_gt, n_images, nc, float(ovthresh), int(bool(use_07_metric)), class_off.data_ptr(),
                                         rec.data_ptr(), prec.data_ptr(), ap.data_ptr(), npos.data_ptr(), status.data_ptr(),
                                         ws.data_ptr(), ws.numel(), _lib.stream_ptr(dev)), "y5obb_dota_eval_f64")
    if dets.present_host is not None:
        present = torch.tensor(dets.present_host, dtype=torch.bool).to(dev, non_blocking=True)
    else:
        present = class_off[1:] > class_off[:-1]
    return Task1Eval(ap, npos, present, class_off, rec, prec, status)
