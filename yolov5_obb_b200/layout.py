"""The model graph as the inference plan (engine.py) and the training plan (train_engine.py) lay it out: module kinds, the
layers a module reads, every layer's output shape, the buffer slice each output lives in, and the stem's space-to-depth
form.  A rule about the graph is written here once, so both plans enforce it."""
from typing import Dict, List, Optional, Tuple

import torch

from .conv import Slice, WindowView


def _kind(m) -> str:
    """Module kind by class NAME, so that the reference's own modules (models/common.py, models/yolo.py,
    torch.nn.Upsample) are accepted as well as the mirrors of yolo.py."""
    return type(m).__name__


def _is(m, name: str) -> bool:
    return _kind(m) == name


def sources(m) -> List[int]:
    """Indices of the layers module m reads: its `f` (parse_model, models/yolo.py:271-323) made absolute."""
    return [m.i - 1 if f == -1 else (f if f >= 0 else m.i + f) for f in ([m.f] if isinstance(m.f, int) else m.f)]


def shapes(layers, H: int, W: int):
    """(ch, hw): output channels and (h, w) of every layer for an H x W input (Detect's entry stays 0, (0, 0))."""
    n = len(layers)
    ch, hw = [0] * n, [(0, 0)] * n
    for m in layers:
        i = m.i
        if _is(m, "Detect"):
            continue
        fs = sources(m)
        in_hw = (H, W) if i == 0 else hw[fs[0]]
        if _is(m, "Conv"):
            s, k, p = m.conv.stride[0], m.conv.kernel_size[0], m.conv.padding[0]
            ch[i] = m.conv.out_channels
            hw[i] = ((in_hw[0] + 2 * p - k) // s + 1, (in_hw[1] + 2 * p - k) // s + 1)
        elif _is(m, "C3"):
            ch[i], hw[i] = m.cv3.conv.out_channels, in_hw
        elif _is(m, "SPPF"):
            ch[i], hw[i] = m.cv2.conv.out_channels, in_hw
        elif _is(m, "Upsample"):
            ch[i], hw[i] = ch[fs[0]], (in_hw[0] * 2, in_hw[1] * 2)
        elif _is(m, "Concat"):
            if any(hw[f] != in_hw for f in fs):
                raise RuntimeError(f"Concat {i} joins inputs of unequal size {[hw[f] for f in fs]}")
            ch[i], hw[i] = sum(ch[f] for f in fs), in_hw
    return ch, hw


def route(layers, ch, hw, new) -> Tuple[List[Optional[Slice]], Dict[int, Slice]]:
    """Where every layer's output lives -> (out, up_of): a Slice per layer (None for Detect), and per Conv followed by an
    nn.Upsample the Concat slice that receives its 2x up-sampled copy (a second store of the Conv's epilogue).  A layer
    feeding a Concat (models/common.py:267-274) stores at its channel offset in the Concat's buffer.
    new(h, w, c) allocates an NHWC buffer; it is called for every Concat's buffer first, then for the other outputs, in
    layer order (the plans' buffer offsets follow that order)."""
    feeds, cat_buf = {}, {}
    for m in layers:
        if _is(m, "Concat"):
            cat_buf[m.i] = new(hw[m.i][0], hw[m.i][1], ch[m.i])
            off = 0
            for s in sources(m):
                if s in feeds:
                    raise RuntimeError("a layer feeding two Concats is not in the shipped yamls")
                feeds[s] = (m.i, off)
                off += ch[s]
    out: List[Optional[Slice]] = [None] * len(layers)
    up_of: Dict[int, Slice] = {}
    for m in layers:
        i = m.i
        if _is(m, "Detect"):
            continue
        if _is(m, "Concat"):
            out[i] = Slice.full(cat_buf[i])
        elif _is(m, "Upsample"):
            if i not in feeds:
                raise RuntimeError("nn.Upsample must feed a Concat (v6.0 head pattern)")
            src = sources(m)[0]
            if not _is(layers[src], "Conv"):
                raise RuntimeError("nn.Upsample must follow a Conv (v6.0 head pattern)")
            j, off = feeds[i]
            out[i] = up_of[src] = Slice(cat_buf[j], off, ch[i])
        elif i in feeds:
            j, off = feeds[i]
            out[i] = Slice(cat_buf[j], off, ch[i])
        else:
            out[i] = Slice.full(new(hw[i][0], hw[i][1], ch[i]))
    return out, up_of


# ---- the stem Conv(3, c, 6, 2, 2) as a 3x1 conv over 48-channel windows of a 2x2 space-to-depth image
def stem_weight(w: torch.Tensor) -> torch.Tensor:
    """[Cout, 3, 6, 6] -> [Cout, 48, 3, 1]: w3[co, tx*16 + (dy*2+dx)*3 + c, ty, 0] = w[co, c, 2ty+dy, 2tx+dx]; channels
    12-15 of every 16 are zero."""
    w2 = torch.zeros((w.shape[0], 16, 3, 3), device=w.device)
    for dy in range(2):
        for dx in range(2):
            w2[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = w[:, :, dy::2, dx::2]
    return w2.permute(0, 3, 1, 2).reshape(w.shape[0], 48, 3, 1).contiguous()


def stem_grad(dw: torch.Tensor, g: torch.Tensor) -> None:
    """The inverse of stem_weight for the weight gradient: dw [ty][Cout][tx*16 + ch16] (the stem wgrad's layout) into the
    parameter gradient g [Cout, 3, 6, 6]."""
    dw = dw.view(3, g.shape[0], 3, 16).permute(1, 3, 0, 2)  # [co, ch16, ty, tx]
    for dy in range(2):
        for dx in range(2):
            g[:, :, dy::2, dx::2].copy_(dw[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3])


def stem_window(x_s2d: torch.Tensor) -> WindowView:
    """The stem's input view of x_s2d [B, H/2, W/2 + 2, 16] (the space-to-depth image with one zero pixel left and right of
    every row): a pixel's three horizontal taps are 48 CONTIGUOUS channels of overlapping windows (pixel stride 16)."""
    B, h, wp, c = x_s2d.shape
    return WindowView(buf=x_s2d, ptr=x_s2d.data_ptr(), pix_stride=c, row_stride=wp * c, img_stride=h * wp * c, B=B, H=h,
                      W=wp - 2, C=3 * c, hbm_c=c)


# ---- which gradients a backward pass computes when some parameters are frozen (train.py --freeze)
def needs_grad(nodes, owns) -> set:
    """The liveness rule: the gradient of a node's output is needed iff the node, or a node upstream of it, owns a
    trainable parameter.  nodes: (node, the nodes it reads) in forward order; owns(node) -> bool."""
    need = set()
    for n, srcs in nodes:
        if owns(n) or any(s in need for s in srcs):
            need.add(n)
    return need


def merge_windows(ranges) -> List[Tuple[int, int]]:
    """Channel ranges [(lo, hi)], sorted, with touching or overlapping ranges joined."""
    out: List[Tuple[int, int]] = []
    for lo, hi in sorted(ranges):
        if out and lo <= out[-1][1]:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


def grad_liveness(layers, ch, trainable):
    """The liveness rule over the model graph.  trainable(m) -> whether layer m owns a trainable parameter.
    Returns (needed, windows): the indices of the layers whose output gradient is needed, and per needed Concat the channel
    windows of its output whose gradient is needed (the slices of its inputs that are in `needed`)."""
    need = needs_grad([(m.i, sources(m) if m.i else []) for m in layers], lambda i: trainable(layers[i]))
    windows = {}
    for m in layers:
        if _is(m, "Concat") and m.i in need:
            off, w = 0, []
            for s in sources(m):
                if s in need:
                    w.append((off, off + ch[s]))
                off += ch[s]
            windows[m.i] = merge_windows(w)
    return need, windows
