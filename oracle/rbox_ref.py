"""numpy/torch-CPU restatement of utils/rboxs_utils.py:9-26,106-165 and
utils/general.py:636-650 — TEST INFRASTRUCTURE.  Pinned by tests/golden/rbox_golden.npz."""
import numpy as np

PI = 3.141592


def gaussian_label_cpu(label, num_class, u=0, sig=4.0):
    x = np.arange(-num_class / 2, num_class / 2)
    y_sig = np.exp(-(x - u) ** 2 / (2 * sig ** 2))
    index = int(num_class / 2 - label)
    return np.concatenate([y_sig[index:], y_sig[:index]], axis=0)


def rbox2poly(obboxes):
    center, w, h, theta = np.split(obboxes.astype(np.float32), (2, 3, 4), axis=-1)
    Cos, Sin = np.cos(theta), np.sin(theta)
    vector1 = np.concatenate([w / 2 * Cos, -w / 2 * Sin], axis=-1)
    vector2 = np.concatenate([-h / 2 * Sin, -h / 2 * Cos], axis=-1)
    point1 = center + vector1 + vector2
    point2 = center + vector1 - vector2
    point3 = center - vector1 - vector2
    point4 = center - vector1 + vector2
    return np.concatenate([point1, point2, point3, point4], axis=-1).reshape(*obboxes.shape[:-1], 8)


def poly2hbb(polys):
    x, y = polys[:, 0::2], polys[:, 1::2]
    x_max, x_min, y_max, y_min = x.max(1), x.min(1), y.max(1), y.min(1)
    return np.stack([(x_max + x_min) / 2.0, (y_max + y_min) / 2.0, x_max - x_min, y_max - y_min], 1)


def scale_polys(img1_shape, polys, img0_shape):
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    polys = polys.copy()
    polys[:, [0, 2, 4, 6]] -= pad[0]
    polys[:, [1, 3, 5, 7]] -= pad[1]
    polys[:, :8] /= gain
    return polys


# ---------------------------------------------------------------------------------------------------------------
# poly2rbox (utils/rboxs_utils.py:39-81).  Its arithmetic is cv2.minAreaRect — a third-party dependency that is not
# of the reference: opencv-python >= 4.5.4 (requirements.txt:6, no lock file).
# Published algorithm (modules/imgproc/src/rotcalipers.cpp): convex hull, then the enclosing rectangle of minimum area
# has a side collinear with a hull edge (rotating calipers); since 4.5.1 the returned angle lies in (0, 90] and `width`
# is the side along that direction.  Restated here edge by edge in float64 and anchored on the reference's own call site
# through tests/golden/p2r_golden.npz (outputs of the REFERENCE function, generated with cv2 4.13.0).
# ---------------------------------------------------------------------------------------------------------------
PI_REF = 3.141592  # utils/rboxs_utils.py:5


def _hull(pts):
    """Andrew's monotone chain; returns the hull vertices (no repeated or collinear points)."""
    p = sorted(set((float(x), float(y)) for x, y in pts))
    if len(p) <= 2:
        return p

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])

    lo, up = [], []
    for q in p:
        while len(lo) >= 2 and cross(lo[-2], lo[-1], q) <= 0:
            lo.pop()
        lo.append(q)
    for q in reversed(p):
        while len(up) >= 2 and cross(up[-2], up[-1], q) <= 0:
            up.pop()
        up.append(q)
    return lo[:-1] + up[:-1]


def min_area_rect(pts):
    """((cx, cy), (w, h), angle_deg) with cv2.minAreaRect's (0, 90] angle convention."""
    h = _hull(pts)
    if len(h) == 1:
        return (h[0][0], h[0][1]), (0.0, 0.0), 0.0
    if len(h) == 2:
        (x0, y0), (x1, y1) = h
        dx, dy = x1 - x0, y1 - y0
        return ((x0 + x1) / 2, (y0 + y1) / 2), (float(np.hypot(dx, dy)), 0.0), float(np.degrees(np.arctan2(dy, dx)))
    P = np.array(h)
    best = None
    for i in range(len(h)):
        e = P[(i + 1) % len(h)] - P[i]
        u = e / np.hypot(*e)
        n = np.array([-u[1], u[0]])
        a, b = P @ u, P @ n
        area = (a.max() - a.min()) * (b.max() - b.min())
        if best is None or area < best[0] * (1 - 1e-12):
            best = (area, u, n, a, b)
    _, u, n, a, b = best
    c = u * (a.max() + a.min()) / 2 + n * (b.max() + b.min()) / 2
    eu, en = a.max() - a.min(), b.max() - b.min()
    alpha = np.degrees(np.arctan2(u[1], u[0])) % 180.0
    if alpha < 1e-9 or alpha > 180.0 - 1e-9:       # horizontal side: the (0, 90] convention names the vertical one `width`
        return (c[0], c[1]), (en, eu), 90.0
    if alpha <= 90.0:
        return (c[0], c[1]), (eu, en), float(alpha)
    return (c[0], c[1]), (en, eu), float(alpha - 90.0)


def regular_theta(theta, start=-PI_REF / 2):  # utils/rboxs_utils.py:28-37, mode '180'
    return (theta - start) % PI_REF + start


def poly2rbox(polys, use_pi=True):
    """utils/rboxs_utils.py:39-81 -> [n, 5] (cx, cy, l, s, theta) with theta in [-pi/2, pi/2) (use_pi) or degrees in [0, 180)."""
    out = []
    for poly in np.asarray(polys, np.float64).reshape(-1, 4, 2):
        (x, y), (w, h), angle = min_area_rect(np.float32(poly).astype(np.float64))
        theta = -angle / 180 * PI_REF
        if w != max(w, h):
            w, h = h, w
            theta += PI_REF / 2
        theta = regular_theta(theta)
        out.append([x, y, w, h, theta if use_pi else theta * 180 / PI_REF + 90])
    return np.array(out)
