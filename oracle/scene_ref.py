"""CPU restatement of the reference's tile-merge chain for whole DOTA scenes — TEST INFRASTRUCTURE for yolov5_obb_b200/scene.py
(never imported by the product package).

Per tile, val.py:50-66 save_one_json keeps round(x, 1) of every polygon coordinate and round(conf, 5) of the score (Python
floats of the fp32 values); tools/TestJson2VocClassTxt.py writes them per class with "%s", which round-trips the doubles;
DOTA_devkit/ResultMerge_multi_process.py:175-236 (mergesingle) shifts each polygon by the tile origin, float(p + left) / 1.0,
runs py_cpu_nms_poly_fast (:62-123, oracle/poly_ref.py) per (scene, class) at nms_thresh and writes
str(round(conf, 2)) / str(round(x, 1)).  Candidates are processed in descending rounded score, ties by lower index
(tile in split order, row): numpy's argsort()[::-1] in the reference orders ties in reverse and is not reproduced."""
import numpy as np

from . import poly_ref


def iou_poly_c(p8, q8):
    """poly_ref.iou_poly with the C division of polyiou.cpp: a zero union (zero-area polygons whose axis-aligned boxes overlap,
    e.g. thin boxes flattened by round(x, 1)) gives nan or +inf there, which suppresses; Python raises instead."""
    try:
        return poly_ref.iou_poly(p8, q8)
    except ZeroDivisionError:
        return float("nan")


def nms_stable(dets, thresh, iou=iou_poly_c):
    """py_cpu_nms_poly_fast with the documented tie rule: the score column is replaced by the rank of the stable descending
    order, which argsort()[::-1] then follows exactly."""
    dets = np.array(dets, np.float64).reshape(-1, 9)
    rank = np.empty(len(dets))
    rank[np.argsort(-dets[:, 8], kind="stable")] = np.arange(len(dets), 0, -1)
    ranked = dets.copy()
    ranked[:, 8] = rank
    return poly_ref.py_cpu_nms_poly_fast(ranked, thresh, iou=iou)


def merge(tiles, nc, thresh=0.2, iou=iou_poly_c):
    """tiles: sequence of (left, up, polys fp32 [n, 8] after scale_polys, conf fp32 [n], cls [n]) in split order ->
    [K, 10] fp64 rows (class, score, x1 y1 ... x4 y4), classes ascending, each class in keep order."""
    per_class = [[] for _ in range(nc)]
    for left, up, polys, conf, cls in tiles:
        polys = np.asarray(polys, np.float32).reshape(-1, 8)
        for p, s, c in zip(polys.tolist(), np.asarray(conf, np.float32).tolist(), np.asarray(cls).tolist()):
            q = [round(x, 1) for x in p]
            det = [float(q[k] + (left if k % 2 == 0 else up)) / float("1") for k in range(8)]
            per_class[int(c)].append(det + [round(s, 5)])
    rows = []
    for c, dets in enumerate(per_class):
        if not dets:
            continue
        for k in nms_stable(dets, thresh, iou):
            rows.append([float(c), dets[k][8]] + dets[k][:8])
    return np.array(rows, np.float64).reshape(-1, 10)


def task1_lines(rows, scene_name, names):
    """{Task1 file name: text} of mergesingle for one scene's merged rows."""
    out = {}
    for r in np.asarray(rows, np.float64).tolist():
        line = scene_name + " " + str(round(r[1], 2)) + " " + " ".join(map(str, [round(x, 1) for x in r[2:]]))
        key = f"Task1_{names[int(r[0])]}.txt"
        out[key] = out.get(key, "") + line + "\n"
    return out
