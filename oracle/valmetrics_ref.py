"""CPU restatement of the validation metrics - TEST INFRASTRUCTURE for yolov5_obb_b200/val.py ValStats / Validator (never
imported by the product package).

* image_stats: the per-image (correct, conf, cls, tcls) entries the reference's val.py:209-250 collects for one batch;
* concat_stats: their concatenation (val.py:268);
* ap_per_class: utils/metrics.py:21-114 with plot=False, also returning the 1000-point p / r curves, with one deliberate
  difference: rows are ordered by a stable argsort of -conf over the input order, so tied confidences keep (image, row)
  order where the reference's np.argsort order for ties is unspecified;
* val_metrics: the val.py:268-276 / 330-332 tail (the stats[0].any() gate, mp, mr, map50, map, maps), and fitness
  (utils/metrics.py:15-18)."""
import numpy as np

EPS = 1e-16
FITNESS_W = [0.0, 0.0, 0.1, 0.9]  # P, R, mAP@0.5, mAP@0.5:0.95

_trapezoid = getattr(np, "trapezoid", None) or np.trapz


def image_stats(correct, dets, counts, targets, niou):
    """correct [B, max_det, niou] bool, dets [B, max_det, 7], counts [B], targets [nt, >= 2] (image, cls, ...) -> the list of
    (correct [n, niou] bool, conf [n] fp32, cls [n] fp32, tcls list of floats) of the images that have detections or labels,
    in image order."""
    out = []
    targets = np.asarray(targets, np.float32)
    targets = targets.reshape(len(targets), -1) if targets.size else np.zeros((0, 2), np.float32)
    for b in range(len(counts)):
        tcls = targets[targets[:, 0] == b, 1].tolist()
        n = int(counts[b])
        if n == 0:
            if tcls:
                out.append((np.zeros((0, niou), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), tcls))
            continue
        c = np.asarray(correct[b, :n], bool) if tcls else np.zeros((n, niou), bool)
        out.append((c, np.asarray(dets[b, :n, 5], np.float32), np.asarray(dets[b, :n, 6], np.float32), tcls))
    return out


def concat_stats(stats):
    """[tp, conf, pred_cls, target_cls] or [] when no image contributed."""
    return [np.concatenate(x, 0) for x in zip(*stats)]


def _compute_ap(recall, precision):
    mrec = np.concatenate(([0.0], recall, [1.0]))
    mpre = np.concatenate(([1.0], precision, [0.0]))
    env = np.maximum.accumulate(mpre[::-1])[::-1]          # the precision envelope
    x = np.linspace(0, 1, 101)
    return _trapezoid(np.interp(x, mrec, env), x)


def ap_per_class(tp, conf, pred_cls, target_cls):
    """-> dict(p_curve, r_curve [n_u, 1000], ap [n_u, niou], ap_class int32, nt int64 [n_u], and tp, fp, p, r, f1 at the
    index of the largest mean F1)."""
    order = np.argsort(-conf, kind="stable")
    tp, conf, pred_cls = tp[order], conf[order], pred_cls[order]
    classes, nt = np.unique(target_cls, return_counts=True)
    px = np.linspace(0, 1, 1000)
    ap = np.zeros((classes.shape[0], tp.shape[1]))
    p, r = np.zeros((classes.shape[0], 1000)), np.zeros((classes.shape[0], 1000))
    for u, c in enumerate(classes):
        sel = pred_cls == c
        if sel.sum() == 0:
            continue
        tpc = tp[sel].cumsum(0)
        fpc = (1 - tp[sel]).cumsum(0)
        recall = tpc / (nt[u] + EPS)
        precision = tpc / (tpc + fpc)
        r[u] = np.interp(-px, -conf[sel], recall[:, 0], left=0)
        p[u] = np.interp(-px, -conf[sel], precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[u, j] = _compute_ap(recall[:, j], precision[:, j])
    f1 = 2 * p * r / (p + r + EPS)
    i = f1.mean(0).argmax()
    pi, ri, f1i = p[:, i], r[:, i], f1[:, i]
    tpi = (ri * nt).round()
    fpi = (tpi / (pi + EPS) - tpi).round()
    return dict(p_curve=p, r_curve=r, ap=ap, ap_class=classes.astype("int32"), nt=nt, tp=tpi, fp=fpi, p=pi, r=ri, f1=f1i)


def val_metrics(stats, nc):
    """stats = concat_stats(...) -> dict(results (mp, mr, map50, map), maps [nc], p, r, ap50, ap, ap_class, curves)."""
    mp = mr = map50 = map_ = 0.0
    out = dict(p=np.zeros(0), r=np.zeros(0), ap50=np.zeros(0), ap=np.zeros(0), ap_class=np.zeros(0, np.int32))
    if len(stats) and stats[0].any():
        res = ap_per_class(*stats)
        ap50, ap = res["ap"][:, 0], res["ap"].mean(1)
        mp, mr, map50, map_ = res["p"].mean(), res["r"].mean(), ap50.mean(), ap.mean()
        out.update(p=res["p"], r=res["r"], ap50=ap50, ap=ap, ap_class=res["ap_class"], curves=res)
    maps = np.zeros(nc) + map_
    for i, c in enumerate(out["ap_class"]):
        maps[c] = out["ap"][i]
    out.update(results=(mp, mr, map50, map_), maps=maps)
    return out


def fitness(x):
    return (x[:, :4] * FITNESS_W).sum(1)
