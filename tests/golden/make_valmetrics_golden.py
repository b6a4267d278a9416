"""Golden vectors for the validation metrics, produced by the REFERENCE's own utils/metrics.py ap_per_class (plot=False) and
fitness on seeded stats with unique confidences (tests/valmetricsgen.py), followed by the val.py:268-276 / 330-332 tail.
The 1000-point p / r curves are the arrays ap_per_class's own np.interp calls return.  The per-image stats val.py:209-250
builds from the valgen batches (process_batch per image) are recorded too.  Only inputs and outputs are stored.
python tests/golden/make_valmetrics_golden.py"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
import val as ref_val  # noqa: E402
import utils.metrics as ref_metrics  # noqa: E402
from utils.general import xywh2xyxy, scale_coords, scale_polys  # noqa: E402
from utils.rboxs_utils import rbox2poly, poly2hbb  # noqa: E402
from tests.valmetricsgen import MIXED, synth_stats, val_batches  # noqa: E402

NC = 8


class _InterpSpy:
    """utils.metrics' numpy with np.interp recorded: the 1000-point calls are ap_per_class's r and p curves, in that order."""

    def __init__(self):
        self.curves = []

    def __getattr__(self, k):
        return getattr(np, k)

    def interp(self, x, *a, **k):
        y = np.interp(x, *a, **k)
        if len(x) == 1000:
            self.curves.append(y)
        return y


def reference_metrics(stats, nc):
    """ap_per_class + fitness of the reference on concatenated stats, with the tail of val.py:268-276 / 330-332."""
    spy = _InterpSpy()
    ref_metrics.np = spy
    out = {}
    mp = mr = map50 = map_ = 0.0
    ap, ap_class = [], []
    if len(stats) and stats[0].any():
        tp, fp, p, r, f1, ap, ap_class = ref_metrics.ap_per_class(*stats, plot=False, names={})
        out.update(tp=tp, fp=fp, p=p, r=r, f1=f1, ap_full=ap, ap_class=ap_class)
        ap50, ap = ap[:, 0], ap.mean(1)
        mp, mr, map50, map_ = p.mean(), r.mean(), ap50.mean(), ap.mean()
        out.update(ap50=ap50, ap=ap)
        # curves of the classes with predictions, in class order; the rest are zero rows
        classes = np.unique(stats[3])
        rc, pc = np.zeros((len(classes), 1000)), np.zeros((len(classes), 1000))
        k = 0
        for u, c in enumerate(classes):
            if (stats[2] == c).sum():
                rc[u], pc[u] = spy.curves[k], spy.curves[k + 1]
                k += 2
        assert k == len(spy.curves)
        out.update(r_curve=rc, p_curve=pc)
    ref_metrics.np = np
    maps = np.zeros(nc) + map_
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    results = (mp, mr, map50, map_)
    out.update(results=np.array(results, np.float64), maps=maps,
               fitness=ref_metrics.fitness(np.array(results).reshape(1, -1)))
    return out


def case_stats():
    cases = {}
    for name, kw in (("mixed10", dict(niou=10, seed=1)), ("mixed1", dict(niou=1, seed=2)),
                     ("notp", dict(niou=10, seed=3, no_tp=True)), ("small", dict(niou=10, seed=4, classes=MIXED[3:5]))):
        tp, conf, cls, tcls, image, row = synth_stats(**kw)
        assert len(np.unique(conf)) == len(conf)
        cases[name] = ([tp, conf, cls, tcls], image, row)
    return cases


def valgen_stats():
    """val.py:209-250 on the valgen batches: one (correct, conf, cls, tcls) entry per image with detections or labels."""
    stats, per_image = [], []
    iouv = torch.linspace(0.5, 0.95, 10)
    for bi, (dets, counts, targets, shapes) in enumerate(val_batches()):
        targets = torch.from_numpy(targets)
        for si in range(dets.shape[0]):
            labels = targets[targets[:, 0] == si, 1:7]
            nl = len(labels)
            tcls = labels[:, 0].tolist() if nl else []
            pred = torch.from_numpy(dets[si, :counts[si]]).clone()
            if len(pred) == 0:
                if nl:
                    stats.append((torch.zeros(0, 10, dtype=torch.bool), torch.Tensor(), torch.Tensor(), tcls))
                    per_image.append((bi, si))
                continue
            poly = rbox2poly(pred[:, :5])
            pred_poly = torch.cat((poly, pred[:, -2:]), dim=1)
            pred_polyn = pred_poly.clone()
            scale_polys((1024, 1024), pred_polyn[:, :8], shapes[si][0], shapes[si][1])
            hbboxn = xywh2xyxy(poly2hbb(pred_polyn[:, :8]))
            pred_hbbn = torch.cat((hbboxn, pred_polyn[:, -2:]), dim=1)
            if nl:
                tbox = xywh2xyxy(poly2hbb(rbox2poly(labels[:, 1:6])))
                scale_coords((1024, 1024), tbox, shapes[si][0], shapes[si][1])
                correct = ref_val.process_batch(pred_hbbn, torch.cat((labels[:, 0:1], tbox), 1), iouv)
            else:
                correct = torch.zeros(pred.shape[0], 10, dtype=torch.bool)
            stats.append((correct.cpu(), pred_poly[:, 8].cpu(), pred_poly[:, 9].cpu(), tcls))
            per_image.append((bi, si))
    return stats, per_image


def main():
    out = {}
    for name, (stats, image, row) in case_stats().items():
        for i, k in enumerate(("tp", "conf", "pred_cls", "target_cls")):
            out[f"{name}/in/{k}"] = stats[i]
        out[f"{name}/in/image"], out[f"{name}/in/row"] = image, row
        for k, v in reference_metrics(stats, NC).items():
            out[f"{name}/{k}"] = np.asarray(v)
        print(name, len(stats[1]), out[f"{name}/results"], out[f"{name}/fitness"])
    stats, per_image = valgen_stats()
    out["valgen/per_image"] = np.array(per_image, np.int64)
    out["valgen/lengths"] = np.array([len(s[1]) for s in stats], np.int64)
    out["valgen/tcls_lengths"] = np.array([len(s[3]) for s in stats], np.int64)
    cat = [np.concatenate(x, 0) for x in zip(*stats)]
    for i, k in enumerate(("tp", "conf", "pred_cls", "target_cls")):
        out[f"valgen/stats/{k}"] = cat[i]
    assert len(np.unique(cat[1])) == len(cat[1]), "valgen confidences tie: the reference's order would be unspecified"
    for k, v in reference_metrics(cat, 15).items():
        out[f"valgen/{k}"] = np.asarray(v)
    print("valgen", len(cat[1]), out["valgen/results"], out["valgen/fitness"])
    np.savez_compressed(HERE / "valmetrics_golden.npz", **out)


if __name__ == "__main__":
    main()
