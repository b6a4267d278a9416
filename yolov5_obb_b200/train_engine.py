"""Training-mode plan: Conv = tensor-core conv (raw) -> batch statistics -> normalise + SiLU, every intermediate
kept for the backward pass.  Mirrors models/yolo.py:163-181 (_forward_once) in train mode
(train.py:324-326): BatchNorm uses batch statistics (eps 1e-3) and updates its running statistics with momentum
0.03 (utils/torch_utils.py:160-162); Detect returns the three raw [B, 3, H, W, no] tensors (yolo.py:62-65,81).

Differences from the inference plan (engine.py): BN is not folded, nothing is updated in place (backward needs
every activation), cv1/cv2 of a C3 run as separate GEMMs (each has its own BatchNorm), and the raw conv output z
of every layer is stored next to its activated output y."""
from typing import Dict, List, Optional

import torch

from . import _lib
from .conv import Conv as ConvOp, Slice, WindowView, pack_weights, MODE_DETECT
from .engine import _is


class _BNLayer:
    """One Conv module in training mode: buffers and launch closures."""

    def __init__(self, mod, x, z: Slice, y: Slice, res: Optional[Slice], y2x: Optional[Slice]):
        self.mod, self.x, self.z, self.y, self.res, self.y2x = mod, x, z, y, res, y2x
        C = z.C
        dev = z.buf.device
        self.sum = torch.zeros(C, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(C, dtype=torch.float32, device=dev)
        self.scale = torch.empty(C, dtype=torch.float32, device=dev)
        self.shift = torch.empty(C, dtype=torch.float32, device=dev)
        self.mean = torch.empty(C, dtype=torch.float32, device=dev)
        self.invstd = torch.empty(C, dtype=torch.float32, device=dev)
        self.conv: Optional[ConvOp] = None
        self.act = isinstance(mod.act, torch.nn.SiLU)


class TrainEngine:
    def __init__(self, model, B: int, H: int, W: int, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("TrainEngine needs a CUDA device (sm_90a); there is no CPU path")
        det = model.model[-1]
        smax = int(max(model.stride))
        if H % smax or W % smax:
            raise RuntimeError(f"image size {H}x{W} must be a multiple of the max stride {smax}")
        self.device, self.B, self.H, self.W = device, B, H, W
        self.model = model
        self.layers: List[_BNLayer] = []
        self.pre_ops, self.keep = [], []
        self.flops = 0.0
        L = _lib.lib()
        self._L = L
        mods = list(model.model)
        n = len(mods)

        def src_of(i, f):
            return i - 1 if f == -1 else (f if f >= 0 else i + f)

        ch, hw = [0] * n, [(0, 0)] * n
        for m in mods:
            i = m.i
            if _is(m, "Detect"):
                continue
            fs = [src_of(i, f) for f in ([m.f] if isinstance(m.f, int) else m.f)]
            in_hw = (H, W) if i == 0 else hw[fs[0]]
            if _is(m, "Conv"):
                s, k, p = m.conv.stride[0], m.conv.kernel_size[0], m.conv.padding[0]
                ch[i], hw[i] = m.conv.out_channels, ((in_hw[0] + 2 * p - k) // s + 1, (in_hw[1] + 2 * p - k) // s + 1)
            elif _is(m, "C3"):
                ch[i], hw[i] = m.cv3.conv.out_channels, in_hw
            elif _is(m, "SPPF"):
                ch[i], hw[i] = m.cv2.conv.out_channels, in_hw
            elif _is(m, "Upsample"):
                ch[i], hw[i] = ch[fs[0]], (in_hw[0] * 2, in_hw[1] * 2)
            elif _is(m, "Concat"):
                ch[i], hw[i] = sum(ch[f] for f in fs), in_hw

        def new(h, w, c):
            t = torch.zeros((B, h, w, c), dtype=torch.bfloat16, device=device)
            self.keep.append(t)
            return t

        feeds, cat_buf = {}, {}
        for m in mods:
            if _is(m, "Concat"):
                cat_buf[m.i] = new(hw[m.i][0], hw[m.i][1], ch[m.i])
                off = 0
                for f in m.f:
                    s = src_of(m.i, f)
                    feeds[s] = (m.i, off)
                    off += ch[s]
        out: List[Optional[Slice]] = [None] * n
        up_of: Dict[int, Slice] = {}
        for m in mods:
            i = m.i
            if _is(m, "Detect"):
                continue
            if _is(m, "Concat"):
                out[i] = Slice.full(cat_buf[i])
            elif _is(m, "Upsample"):
                j, off = feeds[i]
                src = src_of(i, m.f)
                if not _is(mods[src], "Conv"):
                    raise RuntimeError("nn.Upsample must follow a Conv (v6.0 head pattern)")
                up_of[src] = Slice(cat_buf[j], off, ch[i])
                out[i] = up_of[src]
            elif i in feeds:
                j, off = feeds[i]
                out[i] = Slice(cat_buf[j], off, ch[i])
            else:
                out[i] = Slice.full(new(hw[i][0], hw[i][1], ch[i]))

        def add(mod, x, dst: Slice, res=None, y2x=None, stem=False):
            conv = mod.conv
            k, s, p = conv.kernel_size[0], conv.stride[0], conv.padding[0]
            hh, ww = dst.H, dst.W
            z = Slice.full(new(hh, ww, conv.out_channels))
            lay = _BNLayer(mod, x, z, dst, res, y2x)
            w = conv.weight.detach().float()
            if stem:
                w2 = torch.zeros((w.shape[0], 16, 3, 3), device=w.device)
                for dy in range(2):
                    for dx in range(2):
                        w2[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = w[:, :, dy::2, dx::2]
                w = w2.permute(0, 3, 1, 2).reshape(w.shape[0], 48, 3, 1).contiguous()
                wp, bp = pack_weights(w, None)
                lay.conv = ConvOp(x, wp, bp, w.shape[0], (3, 1), 1, (1, 0), False, out=z)
            else:
                wp, bp = pack_weights(w, None)
                lay.conv = ConvOp(x, wp, bp, w.shape[0], k, s, p, False, out=z)
            lay.wp, lay.stem = wp, stem
            self.flops += lay.conv.info()["flops"]
            self.layers.append(lay)
            return lay

        self.x_s2d = torch.zeros((B, H // 2, W // 2 + 2, 16), dtype=torch.bfloat16, device=device)
        self.sppf = None
        for m in mods:
            i = m.i
            if _is(m, "Detect"):
                break
            fs = [src_of(i, f) for f in ([m.f] if isinstance(m.f, int) else m.f)]
            if _is(m, "Conv"):
                if i == 0:
                    Wp = W // 2 + 2
                    win = WindowView(buf=self.x_s2d, ptr=self.x_s2d.data_ptr(), pix_stride=16, row_stride=Wp * 16,
                                     img_stride=(H // 2) * Wp * 16, B=B, H=H // 2, W=W // 2, C=48, hbm_c=16)
                    add(m, win, out[i], stem=True)
                else:
                    add(m, out[fs[0]], out[i], y2x=up_of.get(i))
            elif _is(m, "C3"):
                x = out[fs[0]]
                c_ = m.cv1.conv.out_channels
                hh, ww = hw[i]
                cat = new(hh, ww, 2 * c_)
                cur = Slice.full(new(hh, ww, c_))
                add(m.cv1, x, cur)
                nb = len(m.m)
                for bi, bt in enumerate(m.m):
                    t = Slice.full(new(hh, ww, bt.cv1.conv.out_channels))
                    add(bt.cv1, cur, t)
                    dst = Slice(cat, 0, c_) if bi == nb - 1 else Slice.full(new(hh, ww, c_))
                    add(bt.cv2, t, dst, res=cur if bt.add else None)
                    cur = dst
                add(m.cv2, x, Slice(cat, c_, c_))
                add(m.cv3, Slice.full(cat), out[i])
            elif _is(m, "SPPF"):
                x = out[fs[0]]
                c_ = m.cv1.conv.out_channels
                hh, ww = hw[i]
                cat4 = new(hh, ww, 4 * c_)
                add(m.cv1, x, Slice(cat4, 0, c_))
                self.layers.append(("pool", cat4, hh, ww, c_))
                add(m.cv2, Slice.full(cat4), out[i])

        # Detect: raw logits per level, fp32 [B, na, H, W, no]
        self.det_out, self.det_convs = [], []
        for l, f in enumerate(det.f):
            mi = det.m[l]
            hh, ww = hw[f]
            o = torch.empty((B, det.na, hh, ww, det.no), dtype=torch.float32, device=device)
            wp, bp = pack_weights(mi.weight.detach().float(), mi.bias.detach().float(), MODE_DETECT, det.no)
            stride = float(det.stride[l])
            cv = ConvOp(out[f], wp, bp, mi.weight.shape[0], 1, 1, 0, False,
                        det=dict(out=o, rows_per_image=det.na * hh * ww, row_off=0, no=det.no, decode=False, stride=stride,
                                 anchors_px=(det.anchors[l].detach().float().cpu() * stride).flatten().tolist()))
            self.flops += cv.info()["flops"]
            self.det_out.append(o)
            self.det_convs.append(cv)
        self.out_slices = out
        self._bwd, self._pack, self._pack_has_bwd = None, None, False
        self.prof = None  # set to {} to collect per-kernel-kind device times (ms) during forward()
        import os
        self.use_graph = os.environ.get("Y5OBB_NO_GRAPH", "0") != "1"
        self._graphs = {}
        self._nbt = [lay.mod.bn.num_batches_tracked for lay in self.layers if not isinstance(lay, tuple)]
        cmax = max([lay.z.C for lay in self.layers if not isinstance(lay, tuple)] + [det.na * 256])
        self.scratch = torch.zeros(int(L.y5obb_bn_scratch_floats(cmax)), dtype=torch.float32, device=device)  # reductions

    @staticmethod
    def _stem_weight(w):
        w2 = torch.zeros((w.shape[0], 16, 3, 3), device=w.device)
        for dy in range(2):
            for dx in range(2):
                w2[:, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = w[:, :, dy::2, dx::2]
        return w2.permute(0, 3, 1, 2).reshape(w.shape[0], 48, 3, 1).contiguous()

    def refresh_weights(self):
        """Re-pack the (updated) fp32 parameters into the bf16 buffers the TMA descriptors point at — after every
        optimizer.step().  One launch for all layers, forward and data-gradient layouts (csrc/pack_weights.cu)."""
        if self._pack is None:
            from .train_ops import PackPlan, PACK_FWD, PACK_STEM, PACK_DETECT, PACK_DETECT_BIAS
            det = self.model.model[-1]
            ent = []
            for lay in self.layers:
                if isinstance(lay, tuple):
                    continue
                ent.append((PACK_STEM if lay.stem else PACK_FWD, lay.mod.conv.weight.data, lay.wp, 0, 0))
            for l, cv in enumerate(self.det_convs):
                bn = cv._keep[1].shape[1] // det.na
                ent.append((PACK_DETECT, det.m[l].weight.data, cv._keep[1], det.no, bn))
                ent.append((PACK_DETECT_BIAS, det.m[l].bias.data, cv._keep[2], det.no, bn))
            if self._bwd is not None:
                ent += self._bwd.pack_entries()
            self._pack = PackPlan(ent, self.device)
            self._pack_has_bwd = self._bwd is not None
        self._pack.run()

    def forward(self, x: torch.Tensor, refresh: bool = False):
        """x: [B,3,H,W] fp32 in [0,1] or uint8 -> list of 3 raw prediction tensors [B, na, H_i, W_i, no] fp32.
        refresh=True re-packs the weights from the current parameters first (after an optimizer step).

        The launch sequence is fixed (same buffers every step), so from the third call on it is replayed as ONE CUDA
        graph per input dtype: ~330 launches collapse into a single cudaGraphLaunch (Y5OBB_NO_GRAPH=1 disables)."""
        _lib.require_cuda(x, "x")
        if tuple(x.shape) != (self.B, 3, self.H, self.W):
            raise RuntimeError(f"engine was planned for {(self.B, 3, self.H, self.W)}, got {tuple(x.shape)}")
        if x.dtype != torch.uint8:
            x = x.float()
        if self.prof is not None or not self.use_graph:
            return self._forward_eager(x.contiguous(), refresh)
        slot = self._graphs.setdefault((x.dtype, refresh), dict(calls=0, graph=None, x=None))
        slot["calls"] += 1
        if slot["calls"] == 1:  # first call: eager (warm-up; plans and lazily built state settle)
            return self._forward_eager(x.contiguous(), refresh)
        if slot["graph"] is None:
            if refresh and self._pack is None:
                self.refresh_weights()  # builds the packing plan (allocates): not capturable
            slot["x"] = torch.empty_like(x, memory_format=torch.contiguous_format)
            slot["x"].copy_(x)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self._forward_eager(slot["x"], refresh)
            slot["graph"] = g
        slot["x"].copy_(x)
        slot["graph"].replay()
        return self.det_out

    def _forward_eager(self, x: torch.Tensor, refresh: bool = False):
        if refresh:
            self.refresh_weights()
        L, st = self._L, _lib.stream_ptr(self.device)
        evs = [] if self.prof is not None else None

        def run(tag, rc_fn):
            if evs is None:
                _lib.check(rc_fn(), tag)
                return
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(rc_fn(), tag)
            e1.record()
            evs.append((tag, e0, e1))

        with torch.cuda.device(self.device):
            if x.dtype == torch.uint8:
                run("s2d", lambda: L.y5obb_stem_s2d_u8(x.data_ptr(), self.x_s2d.data_ptr(), self.B, self.H, self.W, 1, st))
            else:
                run("s2d", lambda: L.y5obb_stem_s2d(x.data_ptr(), self.x_s2d.data_ptr(), self.B, self.H, self.W, 1, st))
            for lay in self.layers:
                if isinstance(lay, tuple):
                    _, cat4, hh, ww, c_ = lay
                    run("pool", lambda: L.y5obb_sppf_pool(cat4.data_ptr(), cat4.shape[3], self.B, hh, ww, c_, st))
                    continue
                run("conv", lambda: L.y5obb_conv_run(lay.conv._h, st))
                z, y = lay.z, lay.y
                npix = z.B * z.H * z.W
                bn = lay.mod.bn
                run("bn_stats", lambda: L.y5obb_bn_batch_stats(
                    z.ptr, z.pix_stride, npix, z.C, bn.weight.data_ptr(), bn.bias.data_ptr(), float(bn.eps), float(bn.momentum),
                    bn.running_mean.data_ptr(), bn.running_var.data_ptr(), lay.scale.data_ptr(), lay.shift.data_ptr(),
                    lay.mean.data_ptr(), lay.invstd.data_ptr(), self.scratch.data_ptr(), self.scratch.numel(), st))
                run("bn_apply", lambda: L.y5obb_bn_silu_apply(
                    z.ptr, z.pix_stride, npix, z.C, z.W, lay.scale.data_ptr(), lay.shift.data_ptr(), int(lay.act),
                    lay.res.ptr if lay.res else None, lay.res.pix_stride if lay.res else 0, y.ptr, y.pix_stride,
                    lay.y2x.ptr if lay.y2x else None, lay.y2x.pix_stride if lay.y2x else 0, st))
            for cv in self.det_convs:
                run("detect", lambda: L.y5obb_conv_run(cv._h, st))
            torch._foreach_add_(self._nbt, 1)  # BatchNorm2d.num_batches_tracked of every layer
        if evs is not None:
            torch.cuda.synchronize()
            self.prof = {}
            for tag, e0, e1 in evs:
                self.prof.setdefault(tag, []).append(e0.elapsed_time(e1))
        return self.det_out

    def backward(self, grads):
        """grads: dLoss/d(det_out[l]) for the three levels -> the BackwardPlan, whose .flat holds every parameter
        gradient (fp32, model.parameters() order, see train_backward.py)."""
        if self._bwd is None:
            from .train_backward import BackwardPlan
            self._bwd = BackwardPlan(self)     # packs its data-gradient weights from the current parameters
            self._pack = None                  # the next refresh_weights() covers them too ...
            self._graphs = {}                  # ... so captured forward graphs (old packing plan) are dropped
        self._bwd.run(grads)
        return self._bwd
