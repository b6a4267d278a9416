"""train.py:314-318 (--multi-scale) restated: the size draw and the new shape of an H x W batch.

The reference's `random.randrange(imgsz * 0.5, imgsz * 1.5 + gs)` takes float bounds, which Python 3.12 refuses; Python
3.8-3.11 converted integral floats to int, so `draw_size` passes those ints."""
import math


def draw_size(rng, imgsz, gs):
    return rng.randrange(int(imgsz * 0.5), int(imgsz * 1.5 + gs)) // gs * gs


def new_shape(sz, gs, shape_hw):
    """-> (ns or None when sf == 1, label_ratio or None), expression by expression."""
    sf = sz / max(shape_hw)
    if sf != 1:
        ns = [math.ceil(x * sf / gs) * gs for x in shape_hw]
        label_ratio = float(ns[0]) / shape_hw[0]
        return ns, label_ratio
    return None, None
