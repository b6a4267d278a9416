"""fp32 PyTorch restatement of the reference loss — TEST INFRASTRUCTURE (never imported by the product).

Follows utils/loss.py:93-120 (ComputeLoss.__init__), :122-192 (__call__), :194-275
(build_targets) and utils/metrics.py:201-243 (bbox_iou, CIoU branch), with the one source shim
SURVEY §8(c) lists (clamp bound as int).  Gradients come from torch autograd.  Pinned by
tests/golden/loss_golden.npz = outputs of the REFERENCE ComputeLoss on seeded inputs.
"""
import math

import torch
import torch.nn.functional as F

DEFAULT_HYP = dict(box=0.05, cls=0.5, cls_pw=1.0, obj=1.0, obj_pw=1.0, theta=0.5, theta_pw=1.0, anchor_t=4.0,
                   fl_gamma=0.0, label_smoothing=0.0)  # data/hyps/obb/hyp.finetune_dota.yaml


def scaled_hyp(hyp: dict, nl: int, nc: int, imgsz: int) -> dict:
    """train.py:249-252: gains rescaled to layers / classes / image size before ComputeLoss sees them."""
    h = dict(hyp)
    h["box"] = hyp["box"] * 3. / nl
    h["cls"] = hyp["cls"] * nc / 80. * 3. / nl
    h["obj"] = hyp["obj"] * (imgsz / 640) ** 2 * 3. / nl
    h["theta"] = hyp["theta"] * 3. / nl
    return h


def bbox_ciou(box1, box2, eps=1e-7):
    """metrics.py:201-236 with x1y1x2y2=False, CIoU=True.  box1 [4,n] (pred, transposed), box2 [n,4]."""
    box2 = box2.T
    b1_x1, b1_x2 = box1[0] - box1[2] / 2, box1[0] + box1[2] / 2
    b1_y1, b1_y2 = box1[1] - box1[3] / 2, box1[1] + box1[3] / 2
    b2_x1, b2_x2 = box2[0] - box2[2] / 2, box2[0] + box2[2] / 2
    b2_y1, b2_y2 = box2[1] - box2[3] / 2, box2[1] + box2[3] / 2
    inter = (torch.min(b1_x2, b2_x2) - torch.max(b1_x1, b2_x1)).clamp(0) * \
            (torch.min(b1_y2, b2_y2) - torch.max(b1_y1, b2_y1)).clamp(0)
    w1, h1 = b1_x2 - b1_x1, b1_y2 - b1_y1 + eps
    w2, h2 = b2_x2 - b2_x1, b2_y2 - b2_y1 + eps
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = torch.max(b1_x2, b2_x2) - torch.min(b1_x1, b2_x1)
    ch = torch.max(b1_y2, b2_y2) - torch.min(b1_y1, b2_y1)
    c2 = cw ** 2 + ch ** 2 + eps
    rho2 = ((b2_x1 + b2_x2 - b1_x1 - b1_x2) ** 2 + (b2_y1 + b2_y2 - b1_y1 - b1_y2) ** 2) / 4
    v = (4 / math.pi ** 2) * torch.pow(torch.atan(w2 / h2) - torch.atan(w1 / h1), 2)
    with torch.no_grad():
        alpha = v / (v - iou + (1 + eps))
    return iou - (rho2 / c2 + v * alpha)


def build_targets(p, targets, anchors, stride, anchor_t, na=3):
    """loss.py:194-275.  anchors [nl, na, 2] in grid units; returns per level (b, a, gj, gi), tbox, anch, tcls, tcsl."""
    nt = targets.shape[0]
    tcls, tbox, indices, anch, tcsl = [], [], [], [], []
    dev = targets.device
    ai = torch.arange(na, device=dev).float().view(na, 1).repeat(1, nt)
    targets = torch.cat((targets.repeat(na, 1, 1), ai[:, :, None]), 2)
    g = 0.5
    off = torch.tensor([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], device=dev).float() * g
    for i in range(len(p)):
        a_i = anchors[i]
        fw, fh = float(p[i].shape[3]), float(p[i].shape[2])
        t = targets.clone()
        t[:, :, 2:6] /= stride[i]
        if nt:
            r = t[:, :, 4:6] / a_i[:, None]
            j = torch.max(r, 1 / r).max(2)[0] < anchor_t
            t = t[j]
            gxy = t[:, 2:4]
            gxi = torch.tensor([fw, fh], device=dev) - gxy
            j, k = ((gxy % 1 < g) & (gxy > 1)).T
            l, m = ((gxi % 1 < g) & (gxi > 1)).T
            j = torch.stack((torch.ones_like(j), j, k, l, m))
            t = t.repeat((5, 1, 1))[j]
            offsets = (torch.zeros_like(gxy)[None] + off[:, None])[j]
        else:
            t = targets[0]
            offsets = 0
        b, c = t[:, :2].long().T
        gxy = t[:, 2:4]
        gwh = t[:, 4:6]
        gij = (gxy - offsets).long()
        gi, gj = gij.T
        a = t[:, -1].long()
        indices.append((b, a, gj.clamp(0, int(fh) - 1), gi.clamp(0, int(fw) - 1)))
        tbox.append(torch.cat((gxy - gij, gwh), 1))
        anch.append(a_i[a])
        tcls.append(c)
        tcsl.append(t[:, 7:-1])
    return tcls, tbox, indices, anch, tcsl


def compute_loss(p, targets, anchors, stride, hyp, nc):
    """loss.py:122-192.  p: list of [B, na, H, W, no] tensors (requires_grad for the backward check).
    Returns (loss[1], items[4])."""
    dev, dt = targets.device, p[0].dtype   # fp64 predictions: CIoU, BCE and autograd in fp64, matching still in fp32
    lcls, lbox, lobj, ltheta = (torch.zeros(1, device=dev, dtype=dt) for _ in range(4))
    tcls, tbox, indices, anch, tcsl = build_targets(p, targets, anchors, stride, hyp["anchor_t"], anchors.shape[1])
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    balance = {3: [4.0, 1.0, 0.4]}.get(len(p), [4.0, 1.0, 0.25, 0.06, 0.02])
    pw = lambda k: torch.tensor([hyp[k]], device=dev, dtype=dt)
    for i, pi in enumerate(p):
        b, a, gj, gi = indices[i]
        tobj = torch.zeros_like(pi[..., 0])
        n = b.shape[0]
        if n:
            ps = pi[b, a, gj, gi]
            pxy = ps[:, :2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * anch[i]
            pbox = torch.cat((pxy, pwh), 1)
            iou = bbox_ciou(pbox.T, tbox[i].to(dt))
            lbox = lbox + (1.0 - iou).mean()
            tobj[b, a, gj, gi] = iou.detach().clamp(0).type(tobj.dtype)  # gr = 1.0; sequential last-writer-wins on CPU
            ci = 5 + nc
            if nc > 1:
                t = torch.full_like(ps[:, 5:ci], cn)
                t[range(n), tcls[i]] = cp
                lcls = lcls + F.binary_cross_entropy_with_logits(ps[:, 5:ci], t, pos_weight=pw("cls_pw"))
            ltheta = ltheta + F.binary_cross_entropy_with_logits(ps[:, ci:], tcsl[i].type(ps.dtype), pos_weight=pw("theta_pw"))
        lobj = lobj + F.binary_cross_entropy_with_logits(pi[..., 4], tobj, pos_weight=pw("obj_pw")) * balance[i]
    lbox = lbox * hyp["box"]
    lobj = lobj * hyp["obj"]
    lcls = lcls * hyp["cls"]
    ltheta = ltheta * hyp["theta"]
    bs = p[0].shape[0]
    return (lbox + lobj + lcls + ltheta) * bs, torch.cat((lbox, lobj, lcls, ltheta)).detach()
