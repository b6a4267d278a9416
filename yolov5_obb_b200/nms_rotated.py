"""Host-side mirror of the reference's rotated-NMS operator interface.

Mirrors utils/nms_rotated/nms_rotated_wrapper.py:6-46 (obb_nms) and the pybind module
utils/nms_rotated/src/nms_rotated_ext.cpp:25-59 (nms_rotated_ext.nms_rotated), same
names, argument meaning and error behaviour (RuntimeError on a failing op), but backed by the
device-resident kernels in csrc/nms.cu through the C ABI (include/y5obb.h).
"""
import numpy as np
import torch

from . import _lib


def nms_rotated(dets: torch.Tensor, scores: torch.Tensor, iou_threshold: float, strict_gt: bool = True,
                drop_small: bool = False) -> torch.Tensor:
    """nms_rotated_ext.nms_rotated(dets[N,5], scores[N], thr) -> LongTensor[K] on dets' device.

    Keep indices refer to the caller's order and are listed by descending score (ties: lower index
    first; the reference leaves ties unordered, nms_rotated_cuda.cu:81).  strict_gt=True is the
    reference CUDA rule `IoU > thr` (nms_rotated_cuda.cu:60); False is the CPU rule `>=`
    (nms_rotated_cpu.cpp:55).
    """
    _lib.require_cuda(dets, "dets")
    _lib.require_cuda(scores, "scores")
    if dets.dim() != 2 or dets.size(1) != 5:
        raise RuntimeError(f"dets must be [N,5], got {tuple(dets.shape)}")
    n = dets.size(0)
    if scores.numel() != n:
        raise RuntimeError("dets and scores must have the same length")
    d = dets.detach().contiguous().float()
    s = scores.detach().contiguous().float()
    L = _lib.lib()
    keep = torch.empty(max(n, 1), dtype=torch.int64, device=dets.device)
    nkeep = torch.empty(1, dtype=torch.int64, device=dets.device)
    flags = (_lib.NMS_STRICT_GT if strict_gt else 0) | (_lib.NMS_DROP_SMALL if drop_small else 0)
    with torch.cuda.device(dets.device):
        nbytes = L.y5obb_nms_workspace_bytes(n, 1, n) + 512
        ws = _lib.workspace(nbytes, dets.device, "nms")
        rc = L.y5obb_nms_rotated_f32(_lib.ptr(d), _lib.ptr(s), n, float(iou_threshold), flags, _lib.ptr(keep),
                                     _lib.ptr(nkeep), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dets.device))
    _lib.check(rc, "y5obb_nms_rotated_f32")
    k = int(nkeep.item())  # the op returns a variable-length tensor: one 8-byte read, as any NMS op
    if k < 0:
        raise RuntimeError("y5obb_nms_rotated_f32: internal capacity error")
    return keep[:k]


def nms_rotated_batched(dets: torch.Tensor, scores: torch.Tensor, group_ids: torch.Tensor, n_groups: int,
                        iou_threshold: float, strict_gt: bool = True, max_per_group: int = 0, max_keep: int = 0):
    """Segmented form of nms_rotated: boxes only compete inside their group (image, or class — what the reference obtains
    by adding cls * 4096 to the centres, utils/general.py:849-851, here without touching the coordinates).
    group_ids: int32 [N] in [0, n_groups).  Returns device tensors (keep int64 [N], n_keep int64 [n_groups],
    seg_off int64 [n_groups + 1]): group g's keepers are keep[seg_off[g] : seg_off[g] + n_keep[g]], indices into the
    caller's order, by descending score.  No host synchronisation."""
    _lib.require_cuda(dets, "dets")
    n = dets.size(0)
    d = dets.detach().contiguous().float()
    s = scores.detach().contiguous().float()
    g = group_ids.detach().contiguous().to(torch.int32)
    dev = dets.device
    keep = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    cnt = torch.empty(n_groups, dtype=torch.int64, device=dev)
    off = torch.empty(n_groups + 1, dtype=torch.int64, device=dev)
    mpg = int(max_per_group) if max_per_group > 0 else n
    L = _lib.lib()
    flags = _lib.NMS_STRICT_GT if strict_gt else 0
    with torch.cuda.device(dev):
        ws = _lib.workspace(L.y5obb_nms_workspace_bytes(n, n_groups, mpg), dev, "nms")
        rc = L.y5obb_nms_rotated_batched_f32(_lib.ptr(d), _lib.ptr(s), _lib.ptr(g), n, n_groups, mpg, float(iou_threshold),
                                             flags, int(max_keep), _lib.ptr(keep), _lib.ptr(cnt), _lib.ptr(off),
                                             _lib.ptr(ws), ws.numel(), _lib.stream_ptr(dev))
    _lib.check(rc, "y5obb_nms_rotated_batched_f32")
    return keep, cnt, off


def nms_poly(dets: torch.Tensor, iou_threshold: float) -> torch.Tensor:
    """nms_rotated_ext.nms_poly(dets[N,9], thr) -> LongTensor[K] on dets' device (src/nms_rotated_ext.cpp:42-55 ->
    src/poly_nms_cuda.cu:144-261): polygons (x1 y1 .. x4 y4 score) processed by descending score (ties: lower index first;
    the reference's torch sort leaves them unordered), a polygon dropped when its IoU with an earlier kept one is > thr.
    The reference's own kernel K2 cannot be built on torch >= 1.11 (THC); this one restates its float polygon IoU."""
    _lib.require_cuda(dets, "dets")
    if dets.dim() != 2 or dets.size(1) != 9:
        raise RuntimeError(f"dets must be [N,9], got {tuple(dets.shape)}")
    n = dets.size(0)
    d = dets.detach().contiguous().float()
    keep = torch.empty(max(n, 1), dtype=torch.int64, device=dets.device)
    nkeep = torch.empty(1, dtype=torch.int64, device=dets.device)
    L = _lib.lib()
    with torch.cuda.device(dets.device):
        ws = _lib.workspace(L.y5obb_poly_nms_f32_workspace_bytes(n), dets.device, "poly_nms_f32")
        rc = L.y5obb_poly_nms_f32(_lib.ptr(d), n, float(iou_threshold), 0, _lib.ptr(keep), _lib.ptr(nkeep), _lib.ptr(ws),
                                  ws.numel(), _lib.stream_ptr(dets.device))
    _lib.check(rc, "y5obb_poly_nms_f32")
    return keep[:int(nkeep.item())]


def poly_nms(dets, iou_thr, device_id=None):
    """nms_rotated_wrapper.py:49-67: (dets[inds], inds); CPU input raises NotImplementedError as the reference does."""
    if isinstance(dets, torch.Tensor):
        is_numpy = False
        dets_th = dets
    elif isinstance(dets, np.ndarray):
        is_numpy = True
        device = 'cpu' if device_id is None else f'cuda:{device_id}'
        dets_th = torch.from_numpy(dets).to(device)
    else:
        raise TypeError('dets must be eithr a Tensor or numpy array, '
                        f'but got {type(dets)}')
    if dets_th.device == torch.device('cpu'):
        raise NotImplementedError
    inds = nms_poly(dets_th.float(), iou_thr)
    if is_numpy:
        inds = inds.cpu().numpy()
    return dets[inds, :], inds


class _Ext:
    """Stands in for the pybind module `utils.nms_rotated.nms_rotated_ext`."""
    nms_rotated = staticmethod(lambda dets, scores, thr: nms_rotated(dets, scores, thr))
    nms_poly = staticmethod(nms_poly)


nms_rotated_ext = _Ext()


def obb_nms(dets, scores, iou_thr, device_id=None):
    """RIoU NMS, signature and return values as nms_rotated_wrapper.py:6-46.

    Args:
        dets (tensor/array): (num, [cx cy w h θ]) θ∈[-pi/2, pi/2)
        scores (tensor/array): (num)
        iou_thr (float)
    Returns:
        dets (tensor): (n_nms, [cx cy w h θ]);  inds (tensor): (n_nms) — a CPU int64 tensor on the
        tensor path (as the reference's `ori_inds[inds]` yields), numpy on the numpy path.
    """
    if isinstance(dets, torch.Tensor):
        is_numpy = False
        dets_th = dets
        scores_th = scores
    elif isinstance(dets, np.ndarray):
        is_numpy = True
        device = f"cuda:{0 if device_id is None else device_id}"  # no CPU path here
        dets_th = torch.from_numpy(dets).to(device)
        scores_th = torch.as_tensor(scores).to(device)
    else:
        raise TypeError('dets must be eithr a Tensor or numpy array, '
                        f'but got {type(dets)}')

    if dets_th.numel() == 0:
        inds = dets_th.new_zeros(0, dtype=torch.int64)
    else:
        # the min(w,h) < 0.001 filter of wrapper.py:32-39 runs inside the kernel (Y5OBB_NMS_DROP_SMALL)
        inds = nms_rotated(dets_th, scores_th, iou_thr, strict_gt=True, drop_small=True).cpu()

    if is_numpy:
        inds = inds.cpu().numpy()
    return dets[inds, :], inds


def rbox_iou_pairs(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """IoU of pairs (a[i], b[i]) of (cx,cy,w,h,θ) boxes — single_box_iou_rotated on the device."""
    _lib.require_cuda(a, "a")
    _lib.require_cuda(b, "b")
    a = a.contiguous().float()
    b = b.contiguous().float()
    if a.shape != b.shape or a.dim() != 2 or a.size(1) != 5:
        raise RuntimeError("a and b must both be [N,5]")
    out = torch.empty(a.size(0), dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        rc = _lib.lib().y5obb_rbox_iou_pairs_f32(_lib.ptr(a), _lib.ptr(b), _lib.ptr(out), a.size(0),
                                                 _lib.stream_ptr(a.device))
    _lib.check(rc, "y5obb_rbox_iou_pairs_f32")
    return out
