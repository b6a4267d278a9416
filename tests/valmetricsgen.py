"""Seeded validation stats for the metric tests: synthetic (tp, conf, pred_cls, target_cls) sets with chosen per-class
shapes, and the valgen batches with one image's detections dropped (an image with labels and no detections)."""
import numpy as np

from tests.valgen import synth_val_batch

# per class: (labels, predictions, kind); kind "tp" = every prediction is a TP in every column, "fp" = none is
MIXED = [(50, 300, None), (5, 0, None), (0, 40, None), (3, 1, "tp"), (10, 10, "tp"), (200, 2000, None), (1, 1, "fp"),
         (0, 0, None)]


def synth_stats(classes=MIXED, niou=10, seed=0, n_images=40, conf_levels=None, no_tp=False):
    """-> (tp [n, niou] bool, conf [n] fp32, pred_cls [n] fp32, target_cls [m] fp64, image [n] int64, row [n] int64) with the
    rows in (image, row) order.  No class has more true positives in a column than labels, and a column's TPs are a subset
    of the previous column's.  Confidences are unique, or drawn from `conf_levels` distinct values (ties everywhere)."""
    rng = np.random.default_rng(seed)
    tp, cls, tcls = [], [], []
    for c, (n_l, n_p, kind) in enumerate(classes):
        tcls += [float(c)] * n_l
        t = np.zeros((n_p, niou), bool)
        if kind == "tp" and not no_tp:
            t[:] = True
        elif kind is None and n_l and n_p and not no_tp:
            k = int(rng.integers(0, min(n_l, n_p) + 1))
            t[rng.choice(n_p, k, replace=False), 0] = True
            for j in range(1, niou):
                t[:, j] = t[:, j - 1] & (rng.random(n_p) < 0.85)
        tp.append(t)
        cls += [float(c)] * n_p
    tp, cls = np.concatenate(tp), np.asarray(cls, np.float32)
    n = len(cls)
    if conf_levels is None:
        conf = (rng.permutation(n) + 1).astype(np.float32) / np.float32(n + 1)
    else:
        conf = (rng.integers(1, conf_levels + 1, n) / conf_levels).astype(np.float32)
    perm = rng.permutation(n)
    tp, conf, cls = tp[perm], conf[perm], cls[perm]
    image = np.sort(rng.integers(0, n_images, n))
    row = np.zeros(n, np.int64)
    for i in range(1, n):
        row[i] = row[i - 1] + 1 if image[i] == image[i - 1] else 0
    return tp, conf, cls, np.asarray(rng.permutation(tcls), np.float64), image.astype(np.int64), row


def val_batches():
    """The valgen batches of seeds 0 and 1; in seed 1, image 0 keeps its labels and loses its detections."""
    out = []
    for seed in (0, 1):
        dets, counts, targets, shapes = synth_val_batch(seed)
        if seed == 1:
            counts = counts.copy()
            counts[0] = 0
            dets = dets.copy()
            dets[0] = 0.0
        out.append((dets, counts, targets, shapes))
    return out
