"""Host-side mirror of utils/general.py:772-862 (non_max_suppression_obb) — same signature
and return value; the per-image Python loop, its >= 6 host syncs per image and the N^2/8-byte mask copy are
replaced by one device pipeline (csrc/nms.cu: k_pp_* + batched rotated NMS) and ONE small D2H read of the
per-image counts at the end."""
from typing import List, Optional, Sequence

import torch

from . import _lib

MAX_WH = 4096     # general.py:793
MAX_NMS = 30000   # general.py:794


class DetectRecords:
    """What yolo.Model.detect_records returns: `data` [B, A, rec_w] fp32 rows (cx, cy, w, h, obj, cls[nc], theta index, pad)
    written by the Detect epilogue (engine-owned buffer, overwritten by the next forward), and the class count.  The theta index
    is the first maximum of the row's 180 theta logits, i.e. what torch.max returns on their sigmoids (utils/general.py:822)."""

    def __init__(self, data: torch.Tensor, nc: int):
        self.data, self.nc = data, int(nc)


def non_max_suppression_obb(prediction: torch.Tensor, conf_thres: float = 0.25, iou_thres: float = 0.45,
                            classes: Optional[Sequence[int]] = None, agnostic: bool = False, multi_label: bool = False,
                            labels=(), max_det: int = 1500, return_packed: bool = False):
    """Runs Non-Maximum Suppression (NMS) on inference results_obb.

    Args:
        prediction (tensor): (b, n_all_anchors, [cx cy l s obj num_cls theta_cls]) fp32 on a CUDA device
    Returns:
        list of detections, len=batch_size, on (n,7) tensor per image [xylsθ, conf, cls] θ ∈ [-pi/2, pi/2)
    """
    compact = isinstance(prediction, DetectRecords)
    if compact:
        nc_rec = prediction.nc
        prediction = prediction.data
    _lib.require_cuda(prediction, "prediction")
    if prediction.dim() != 3:
        raise RuntimeError("prediction must be [batch, anchors, nc+185]")
    nc = nc_rec if compact else prediction.shape[2] - 5 - 180
    assert 0 <= conf_thres <= 1, f'Invalid Confidence threshold {conf_thres}, valid values are between 0.0 and 1.0'
    assert 0 <= iou_thres <= 1, f'Invalid IoU {iou_thres}, valid values are between 0.0 and 1.0'
    if labels:
        raise RuntimeError("apriori `labels` (autolabelling) are not part of the hot path")
    if nc < 1 or nc > 64:
        raise RuntimeError(f"nc={nc} unsupported (1..64)")
    B, A, no = prediction.shape
    if compact:
        no = nc + 185
    dev = prediction.device
    if B == 0 or A == 0:
        return [torch.zeros((0, 7), device=dev) for _ in range(B)]
    pred = prediction.detach().float().contiguous()  # half inputs are widened (the arithmetic is defined in fp32)
    mask = (1 << 64) - 1
    if classes is not None:
        mask = 0
        for c in classes:
            mask |= 1 << int(c)
    worst = B * A * (nc if (multi_label and nc > 1) else 1)
    # optimistic capacity (every kernel of the pipeline runs over `cap` slots); grown on overflow below
    cap = min(worst, max(B * 8192, 1 << 16, int(_CAP_HINT.get((B, A, nc), 0))))
    nosplit = _NO_SPLIT.get((B, A, nc), False)
    args = (pred, B, A, no, nc, conf_thres, iou_thres, mask, agnostic, multi_label, max_det, nosplit, compact)
    if return_packed == "async":
        # no host read at all: (device [B, max_det, 7], device int64 [B + 1] = rows per image + total candidates, cap).
        # The caller checks counts[B] <= cap when it reads the counts (pipeline.DetectPipeline does, and re-runs).
        # Every launch of the pipeline has a fixed geometry (sized by `cap`), so for a fixed input buffer the whole
        # post-process is replayed as ONE CUDA graph from the third identical call on; the two returned tensors are
        # then the graph's static outputs (valid until the next call with the same arguments).
        out, counts = _launch_graphed(args, cap)
        return out, counts, cap
    while True:
        out, counts = _launch(args, cap)
        c = counts.tolist()  # the one host read: rows per image (+ total candidates)
        if c[B] == -2:  # a box reaches another class's offset copy: the class-split shortcut is not exact here
            _NO_SPLIT[(B, A, nc)] = True
            args = args[:-2] + (True, args[-1])
            continue
        if c[B] <= cap:
            break
        cap = min(worst, max(c[B], cap * 4))  # rare: more candidates than the optimistic capacity
        _CAP_HINT[(B, A, nc)] = cap
    if any(k < 0 for k in c[:B]):
        raise RuntimeError("y5obb_nms_obb_f32: internal capacity error")
    if return_packed:  # (device [B, max_det, 7], per-image row counts) — one buffer for a single D2H copy
        return out, c[:B]
    return [out[b, :c[b]] for b in range(B)]


_NO_SPLIT = {}  # (B, anchors, nc) -> True once a batch needed the one-pass-per-image form (sticky)
_CAP_HINT = {}  # (B, anchors, nc) -> candidate capacity that was needed once (sticky: avoids repeated overflow re-runs)


_GRAPHS = {}


def _launch_graphed(args, cap):
    import os
    pred = args[0]
    if os.environ.get("Y5OBB_NO_GRAPH", "0") == "1":
        return _launch(args, cap)
    key = (pred.data_ptr(), pred.device.index, cap) + tuple(args[1:])  # (includes the compact-record flag)
    slot = _GRAPHS.get(key)
    if slot is None:
        if len(_GRAPHS) > 16:
            _GRAPHS.clear()
        slot = _GRAPHS[key] = dict(calls=0, graph=None, out=None, counts=None, ws=None)
    slot["calls"] += 1
    if slot["calls"] <= 2:
        return _launch(args, cap)
    if slot["graph"] is None:
        torch.cuda.synchronize(pred.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            out, counts, ws = _launch(args, cap, keep_ws=True)
        slot.update(graph=g, out=out, counts=counts, ws=ws)
    slot["graph"].replay()
    return slot["out"], slot["counts"]


def _launch(args, cap, keep_ws=False):
    pred, B, A, no, nc, conf_thres, iou_thres, mask, agnostic, multi_label, max_det, nosplit, compact = args
    L = _lib.lib()
    dev = pred.device
    out = torch.empty((B, max_det, 7), dtype=torch.float32, device=dev)
    counts = torch.empty(B + 1, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        nbytes = L.y5obb_nms_obb_workspace_bytes(B, A, cap, MAX_NMS)
        # a captured graph owns its workspace (the shared grow-only buffer may be re-allocated later)
        # (the shared grow-only buffer is per stream: calls on different streams may be in flight together)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev) if keep_ws else \
            _lib.workspace(nbytes, dev, f"nms_obb:{_lib.stream_ptr(dev)}")
        rc = L.y5obb_nms_obb_f32(pred.data_ptr(), B, A, no, nc, float(conf_thres), float(iou_thres), mask,
                                 int(bool(agnostic)), int(bool(multi_label)), int(max_det), MAX_NMS, float(MAX_WH),
                                 _lib.NMS_STRICT_GT | (_lib.NMS_NO_CLASS_SPLIT if nosplit else 0) | (_lib.NMS_COMPACT_PRED if compact else 0),
                                 cap, out.data_ptr(),
                                 counts.data_ptr(), ws.data_ptr(),
                                 ws.numel(), _lib.stream_ptr(dev))
    _lib.check(rc, "y5obb_nms_obb_f32")
    return (out, counts, ws) if keep_ws else (out, counts)
