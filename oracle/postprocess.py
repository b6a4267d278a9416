"""CPU restatement of utils/general.py:772-862 (non_max_suppression_obb) —
TEST INFRASTRUCTURE.  torch CPU ops for the filtering, the pinned C++ oracle for the rotated NMS
(mode 1 = reference CUDA rule `>`, mode 0 = reference CPU rule `>=`).  Pinned by
tests/golden/postprocess_golden.npz (outputs of the reference function itself)."""
import numpy as np
import torch

from . import obb_nms as _oracle_obb_nms

PI = 3.141592  # utils/rboxs_utils.py:5 (general.py imports it)


def ref_obb_nms_cuda(ref):
    """nms_rotated_wrapper.py:6-46 (obb_nms) over the reference's own CUDA kernel K1 (`ref` = oracle/_ref extension,
    oracle.build_ref.load_ref()): too-small filter, kernel, indices mapped back.  For the eager-PyTorch-on-GPU bar."""
    def fn(rboxes, scores, thr):
        too_small = rboxes[:, 2:4].min(1)[0] < 0.001
        if too_small.all():
            return torch.zeros(0, dtype=torch.int64, device=rboxes.device)
        ori = torch.arange(rboxes.shape[0], device=rboxes.device)[~too_small]
        return ori[ref.nms_rotated_cuda(rboxes[~too_small].contiguous(), scores[~too_small].contiguous(), float(thr))]
    return fn


def non_max_suppression_obb(prediction, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
                            multi_label=False, max_det=1500, nms_mode=1, nms_fn=None):
    """nms_fn=None: CPU, the pinned C++ oracle NMS.  nms_fn=callable(rboxes[n,5], scores[n], thr) -> keep indices: the
    same per-image loop on the tensors' own device (e.g. ref_obb_nms_cuda for the eager GPU baseline of bench.py)."""
    prediction = prediction.detach().float()
    if nms_fn is None:
        prediction = prediction.cpu()
    nc = prediction.shape[2] - 5 - 180
    xc = prediction[..., 4] > conf_thres
    class_index = nc + 5
    max_wh, max_nms = 4096, 30000
    multi_label &= nc > 1
    output = [torch.zeros((0, 7), device=prediction.device)] * prediction.shape[0]
    for xi, x in enumerate(prediction):
        x = x[xc[xi]].clone()
        if not x.shape[0]:
            continue
        x[:, 5:class_index] *= x[:, 4:5]
        _, theta_pred = torch.max(x[:, class_index:], 1, keepdim=True)
        theta_pred = (theta_pred - 90) / 180 * PI
        if multi_label:
            i, j = (x[:, 5:class_index] > conf_thres).nonzero(as_tuple=False).T
            x = torch.cat((x[i, :4], theta_pred[i], x[i, j + 5, None], j[:, None].float()), 1)
        else:
            conf, j = x[:, 5:class_index].max(1, keepdim=True)
            x = torch.cat((x[:, :4], theta_pred, conf, j.float()), 1)[conf.view(-1) > conf_thres]
        if classes is not None:
            x = x[(x[:, 6:7] == torch.tensor(classes, device=x.device)).any(1)]
        n = x.shape[0]
        if not n:
            continue
        elif n > max_nms:
            x = x[x[:, 5].argsort(descending=True, stable=True)[:max_nms]]
        c = x[:, 6:7] * (0 if agnostic else max_wh)
        rboxes = x[:, :5].clone()
        rboxes[:, :2] = rboxes[:, :2] + c
        if nms_fn is None:
            keep = torch.from_numpy(_oracle_obb_nms(rboxes.numpy(), x[:, 5].numpy(), float(np.float32(iou_thres)), mode=nms_mode))
        else:
            keep = nms_fn(rboxes, x[:, 5], iou_thres)
        if keep.shape[0] > max_det:
            keep = keep[:max_det]
        output[xi] = x[keep]
    return output
