"""Polygon IoU and the tile-merge polygon NMS of the DOTA devkit — TEST INFRASTRUCTURE for SURVEY section 8f rank 4
(never imported by the product package).

Follows DOTA_devkit/polyiou.cpp:9-128 (iou_poly: the signed-triangle-fan intersection area of two
quadrilaterals, eps = 1e-8 sign test) and DOTA_devkit/ResultMerge_multi_process.py:62-123
(py_cpu_nms_poly_fast: greedy NMS in descending score with an axis-aligned pre-filter whose areas use the +1 pixel
convention while the intersection does not).  Pinned against the reference's own polyiou.cpp compiled in place
(oracle/_ref/libref_polyiou.so, oracle/build_ref.py) and tests/golden/poly_golden.npz."""
import numpy as np

EPS = 1e-8


def _sig(d):
    return (d > EPS) - (d < -EPS)


def _cross(o, a, b):
    return (a[0] - o[0]) * (b[1] - o[1]) - (b[0] - o[0]) * (a[1] - o[1])


def _area(ps):
    n = len(ps)
    res = 0.0
    for i in range(n):
        j = (i + 1) % n
        res += ps[i][0] * ps[j][1] - ps[i][1] * ps[j][0]
    return res / 2.0


def _line_cross(a, b, c, d):
    s1, s2 = _cross(a, b, c), _cross(a, b, d)
    if _sig(s1) == 0 and _sig(s2) == 0:
        return 2, None
    if _sig(s2 - s1) == 0:
        return 0, None
    return 1, ((c[0] * s2 - d[0] * s1) / (s2 - s1), (c[1] * s2 - d[1] * s1) / (s2 - s1))


def _same(p, q):
    return _sig(p[0] - q[0]) == 0 and _sig(p[1] - q[1]) == 0


def _polygon_cut(p, a, b):
    """polyiou.cpp:57-70: keep the part of polygon p to the left of the line a->b."""
    n = len(p)
    pp = []
    for i in range(n):
        pi, pj = p[i], p[(i + 1) % n]
        if _sig(_cross(a, b, pi)) > 0:
            pp.append(pi)
        if _sig(_cross(a, b, pi)) != _sig(_cross(a, b, pj)):
            kind, x = _line_cross(a, b, pi, pj)
            # (lineCross leaves the output point untouched when it returns 0 / 2: the C code then appends whatever the
            # slot held; with sign(cross) differing the lines are not parallel, so kind == 1 here)
            pp.append(x if kind == 1 else pi)
    out = []
    for i, q in enumerate(pp):
        if i == 0 or not _same(q, pp[i - 1]):
            out.append(q)
    while len(out) > 1 and _same(out[-1], out[0]):
        out.pop()
    return out


def _tri_intersect(a, b, c, d):
    """polyiou.cpp:73-88: signed intersection area of triangles (o,a,b) and (o,c,d), o the origin."""
    o = (0.0, 0.0)
    s1, s2 = _sig(_cross(o, a, b)), _sig(_cross(o, c, d))
    if s1 == 0 or s2 == 0:
        return 0.0
    if s1 == -1:
        a, b = b, a
    if s2 == -1:
        c, d = d, c
    p = [o, a, b]
    p = _polygon_cut(p, o, c)
    p = _polygon_cut(p, c, d)
    p = _polygon_cut(p, d, o)
    res = abs(_area(p)) if p else 0.0
    return -res if s1 * s2 == -1 else res


def iou_poly(p8, q8):
    """polyiou.cpp:106-128 on two 8-float polygons (x1 y1 ... x4 y4)."""
    ps1 = [(float(p8[2 * i]), float(p8[2 * i + 1])) for i in range(4)]
    ps2 = [(float(q8[2 * i]), float(q8[2 * i + 1])) for i in range(4)]
    if _area(ps1) < 0:
        ps1.reverse()
    if _area(ps2) < 0:
        ps2.reverse()
    inter = 0.0
    for i in range(4):
        for j in range(4):
            inter += _tri_intersect(ps1[i], ps1[(i + 1) % 4], ps2[j], ps2[(j + 1) % 4])
    union = abs(_area(ps1)) + abs(_area(ps2)) - inter
    return inter / union


def py_cpu_nms_poly_fast(dets, thresh, iou=iou_poly):
    """ResultMerge_multi_process.py:62-123.  dets [n, 9] = 8 polygon coordinates + score -> list of kept indices."""
    dets = np.asarray(dets, np.float64)
    obbs = dets[:, :8]
    x1, y1 = obbs[:, 0::2].min(1), obbs[:, 1::2].min(1)
    x2, y2 = obbs[:, 0::2].max(1), obbs[:, 1::2].max(1)
    areas = (x2 - x1 + 1) * (y2 - y1 + 1)
    order = dets[:, 8].argsort()[::-1]
    keep = []
    while order.size > 0:
        i = order[0]
        keep.append(int(i))
        rest = order[1:]
        w = np.maximum(0.0, np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]))
        h = np.maximum(0.0, np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]))
        hbb_inter = w * h
        ovr = hbb_inter / (areas[i] + areas[rest] - hbb_inter)
        for j in np.where(ovr > 0)[0]:
            ovr[j] = iou(obbs[i], obbs[rest[j]])
        order = rest[np.where(ovr <= thresh)[0]]
    return keep
