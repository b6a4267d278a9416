"""Seeded per-tile detections for the tile-merge tests (tests/test_scene_*.py, tests/golden/make_scene_golden.py).

Objects live in scene coordinates; every tile that contains an object's centre reports it (objects in the 200 px overlaps
appear in two or four tiles with slightly different boxes), in tile-network coordinates (+ the letterbox pad).  Centres and
sizes are multiples of 0.25 px and theta = 0 for the `ties` share, so that polygon coordinates land on exact rounding ties of
round(x, 1) (x.25, x.75) and rbox2poly is exact on any device.  Rounded scores (1e-5) are unique within a class."""
import numpy as np

from yolov5_obb_b200.scene import split_origins


def tile_rows(H, W, n_obj, nc=15, seed=0, subsize=1024, gap=200, pad=16.0, ties=0.5, max_det=1500, rotated=True):
    """-> origins [T, 2] int32, rows [T, max_det, 7] fp32 (cx, cy, l, s, theta, conf, cls), counts [T] int64."""
    rng = np.random.default_rng(seed)
    origins = np.array(split_origins(H, W, subsize, gap), np.int32)
    T = len(origins)
    cx = np.round(rng.uniform(0, W, n_obj) * 4) / 4
    cy = np.round(rng.uniform(0, H, n_obj) * 4) / 4
    l = np.round(rng.uniform(8, 120, n_obj) * 4) / 4
    s = np.round(l * rng.uniform(0.2, 1.0, n_obj) * 4) / 4
    th = np.where(rng.random(n_obj) < ties, 0.0, rng.uniform(-np.pi / 2, np.pi / 2, n_obj) if rotated else 0.0)
    cls = rng.integers(0, nc, n_obj)
    rows = np.zeros((T, max_det, 7), np.float32)
    counts = np.zeros(T, np.int64)
    for t, (left, up) in enumerate(origins):
        inside = np.where((cx >= left) & (cx < left + subsize) & (cy >= up) & (cy < up + subsize))[0]
        inside = inside[:max_det]
        n = len(inside)
        jit = np.round(rng.normal(0, 1.0, (n, 4)) * 4) / 4 * (t > 0)  # the same object differs a little between tiles
        r = rows[t, :n]
        r[:, 0] = cx[inside] - left + pad + jit[:, 0]
        r[:, 1] = cy[inside] - up + pad + jit[:, 1]
        r[:, 2] = np.maximum(l[inside] + jit[:, 2], 2.0)
        r[:, 3] = np.maximum(s[inside] + jit[:, 3], 1.0)
        r[:, 4] = th[inside]
        r[:, 6] = cls[inside]
        counts[t] = n
    # every row its own rounded score k / 1e5 (k unique over the scene), plus a fraction that rounds back to k
    k = rng.choice(np.arange(1000, 100000), size=int(counts.sum()), replace=False)
    o = 0
    for t in range(T):
        n = counts[t]
        rows[t, :n, 5] = ((k[o:o + n] + rng.uniform(-0.3, 0.3, n)) * 1e-5).astype(np.float32)
        o += n
    return origins, rows, counts
