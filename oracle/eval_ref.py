"""CPU restatement of DOTA Task1 evaluation — TEST INFRASTRUCTURE for yolov5_obb_b200/dota_eval.py (never imported by the
product package).

DOTA_devkit/dota_evaluation_task1.py:88-249 voc_eval per class: detections in descending score, each compared with the GTs of
its image and class through the axis-aligned pre-filter (:180-206, +1 pixel convention on the intersection and on both areas
of the union) and polyiou's iou_poly(GT, det) (:212; scene_ref.iou_poly_c, C division), the sequential R['det'] loop
(:223-231), cumulative tp / fp, rec and prec; :54-85 voc_ap with np.add.reduce's pairwise summation written out
(pairwise_sum).  The one deliberate difference: tied scores keep input order (a stable argsort), where the reference's
np.argsort(-confidence) order for ties depends on numpy's version and the host CPU."""
import numpy as np

from .scene_ref import iou_poly_c


def pairwise_sum(v):
    """np.add.reduce of a contiguous fp64 vector: below 8 elements a plain sum from 0.0, up to 128 elements 8 partial sums
    combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) plus the remainder, above that the halves split at n / 2
    rounded down to a multiple of 8."""
    v = [float(x) for x in v]

    def rec(lo, n):
        if n < 8:
            r = 0.0
            for i in range(lo, lo + n):
                r += v[i]
            return r
        if n <= 128:
            r = v[lo:lo + 8]
            i = 8
            while i < n - n % 8:
                for j in range(8):
                    r[j] += v[lo + i + j]
                i += 8
            res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
            for k in range(i, n):
                res += v[lo + k]
            return res
        n2 = n // 2
        n2 -= n2 % 8
        return rec(lo, n2) + rec(lo + n2, n - n2)

    return rec(0, len(v))


def voc_ap(rec, prec, use_07_metric):
    rec, prec = np.asarray(rec, np.float64), np.asarray(prec, np.float64)
    if use_07_metric:
        ap = 0.0
        for t in np.arange(0., 1.1, 0.1):
            sel = prec[rec >= t]
            ap = ap + (float(sel.max()) if sel.size else 0.0) / 11.
        return ap
    mrec = np.concatenate(([0.], rec, [1.]))
    mpre = np.concatenate(([0.], prec, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]   # the suffix-max envelope (max is exact in any order)
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return pairwise_sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def _match(bb, BBGT):
    """(ovmax, jmax) of one detection against the GTs of its image and class."""
    if BBGT.shape[0] == 0:
        return -np.inf, -1
    gx0, gy0 = BBGT[:, 0::2].min(1), BBGT[:, 1::2].min(1)
    gx1, gy1 = BBGT[:, 0::2].max(1), BBGT[:, 1::2].max(1)
    bx0, by0, bx1, by1 = bb[0::2].min(), bb[1::2].min(), bb[0::2].max(), bb[1::2].max()
    iw = np.maximum(np.minimum(gx1, bx1) - np.maximum(gx0, bx0) + 1., 0.)
    ih = np.maximum(np.minimum(gy1, by1) - np.maximum(gy0, by0) + 1., 0.)
    inters = iw * ih
    uni = (bx1 - bx0 + 1.) * (by1 - by0 + 1.) + (gx1 - gx0 + 1.) * (gy1 - gy0 + 1.) - inters
    keep = np.where(inters / uni > 0)[0]
    if keep.size == 0:
        return -np.inf, -1
    ovs = np.array([iou_poly_c(BBGT[j], bb) for j in keep], np.float64)
    return float(np.max(ovs)), int(keep[np.argmax(ovs)])


def evaluate(det_img, det10, gt_img, gt10, nc, ovthresh=0.5, use_07_metric=True):
    """det10 [n, 10] (class, score, 8 coordinates) + det_img [n], gt10 [m, 10] (class, difficult, 8 coordinates) + gt_img [m]
    -> dict(class_off [nc + 1], rec [n], prec [n] (class segments in sorted order), ap [nc], npos [nc])."""
    det_img, det10 = np.asarray(det_img, np.int64), np.asarray(det10, np.float64).reshape(-1, 10)
    gt_img, gt10 = np.asarray(gt_img, np.int64), np.asarray(gt10, np.float64).reshape(-1, 10)
    off, recs, precs, aps, nposs = [0], [], [], [], []
    for c in range(nc):
        gsel = gt10[:, 0] == c
        npos = int((gt10[gsel, 1] == 0).sum())
        recs_c = {}
        for img in np.unique(gt_img[gsel]).tolist():
            g = gt10[gsel & (gt_img == img)]
            recs_c[img] = (g[:, 2:], g[:, 1] != 0, [False] * g.shape[0])
        empty = (np.zeros((0, 8)), np.zeros(0, bool), [])
        sel = np.where(det10[:, 0] == c)[0]
        order = sel[np.argsort(-det10[sel, 1], kind="stable")]
        tp, fp = np.zeros(len(order)), np.zeros(len(order))
        for d, k in enumerate(order.tolist()):
            BBGT, difficult, seen = recs_c.get(int(det_img[k]), empty)
            ovmax, jmax = _match(det10[k, 2:], BBGT)
            if ovmax > ovthresh:
                if not difficult[jmax]:
                    if not seen[jmax]:
                        tp[d] = 1.
                        seen[jmax] = True
                    else:
                        fp[d] = 1.
            else:
                fp[d] = 1.
        tp, fp = np.cumsum(tp), np.cumsum(fp)
        with np.errstate(divide="ignore", invalid="ignore"):
            rec = tp / float(npos)
        prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
        off.append(off[-1] + len(order))
        recs.append(rec)
        precs.append(prec)
        with np.errstate(invalid="ignore"):
            aps.append(voc_ap(rec, prec, use_07_metric))
        nposs.append(npos)
    return dict(class_off=np.array(off, np.int64), rec=np.concatenate(recs), prec=np.concatenate(precs),
                ap=np.array(aps, np.float64), npos=np.array(nposs, np.int64))


def main_map(ap, present):
    """dota_evaluation_task1.py:305-343 main(): the sum of the APs of the classes that have a Task1 file, in class order,
    divided by their number."""
    m, n = 0.0, 0
    for a, p in zip(np.asarray(ap, np.float64).tolist(), present):
        if p:
            m = m + a
            n += 1
    return m / n if n else float("nan")
