"""Training-mode plan: Conv = tensor-core conv (raw) -> batch statistics -> normalise + SiLU, every intermediate
kept for the backward pass.  Mirrors models/yolo.py:163-181 (_forward_once) in train mode
(train.py:324-326): BatchNorm uses batch statistics (eps 1e-3) and updates its running statistics with momentum
0.03 (utils/torch_utils.py:160-162); Detect returns the three raw [B, 3, H, W, no] tensors (yolo.py:62-65,81).

Differences from the inference plan (engine.py): BN is not folded, nothing is updated in place (backward needs
every activation), cv1/cv2 of a C3 run as separate GEMMs (each has its own BatchNorm), and the raw conv output z
of every layer is stored next to its activated output y."""
import weakref
from typing import List, NamedTuple, Optional, Union

import torch

from . import _lib
from .conv import Conv as ConvOp, Slice, pack_weights, MODE_DETECT
from .general import require_nc
from .layout import _is, route, shapes, sources, stem_weight, stem_window


def flat_layout(params):
    """Offsets of every parameter's gradient in the flat fp32 buffer (16-byte aligned views) and its length."""
    offsets, n = [], 0
    for p in params:
        offsets.append(n)
        n += (p.numel() + 3) // 4 * 4
    return offsets, n


class TrainArena:
    """One device allocation that every training plan of a model carves its activation, raw-output, Detect-logit and
    gradient buffers from (Model.reserve_train_arena), plus the one flat parameter-gradient buffer all plans share.

    Plans of different shapes alias the same bytes: only one plan runs at a time, on one stream (the backward's wgrad
    stream joins it before the backward returns).  `owner` is the plan whose data the arena holds; a plan that runs after
    another one re-zeroes the few regions it relies on being zero (TrainEngine.zero_regions) before its first launch."""

    ALIGN = 256

    def __init__(self, nbytes: int, n_flat: int, device):
        self.device = torch.device(device)
        self.buf = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        self.flat = torch.zeros(n_flat, dtype=torch.float32, device=self.device)
        self.owner = None   # weak reference to the TrainEngine whose data the arena holds
        self.last_grad_flat = None   # the clone of the flat gradient the last backward handed to autograd
        self._inputs = {}

    @property
    def nbytes(self) -> int:
        return self.buf.numel()

    def input_buffer(self, shape, dtype) -> torch.Tensor:
        """The static input of the captured forward graphs, one per (shape, dtype) for all plans."""
        key = (tuple(shape), dtype)
        t = self._inputs.get(key)
        if t is None:
            t = self._inputs[key] = torch.empty(key[0], dtype=dtype, device=self.device)
        return t


class _Carver:
    """Bump allocator over a TrainArena (arena=None: ordinary zero-filled allocations whose arena offsets are still
    counted, which is how Model.reserve_train_arena sizes the arena)."""

    def __init__(self, arena: Optional[TrainArena], device):
        self.arena, self.device, self.off = arena, device, 0
        self.zero = []   # regions the plan relies on being zero

    def take(self, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        a = TrainArena.ALIGN
        off = (self.off + a - 1) // a * a
        self.off = off + nbytes
        if self.arena is None:
            return torch.zeros(tuple(shape), dtype=dtype, device=self.device)
        if self.off > self.arena.nbytes:
            raise RuntimeError(f"training plan needs more than the {self.arena.nbytes} bytes of the reserved arena: "
                               "reserve it for the largest batch and image size (Model.reserve_train_arena)")
        return self.arena.buf[off:off + nbytes].view(dtype).view(tuple(shape))

    def zeroed(self, t: torch.Tensor):
        """Register a view of an arena buffer that must read as zero whenever the plan runs (and zero it now)."""
        if self.arena is not None:
            t.zero_()
            self.zero.append(t)


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


class _PoolLayer(NamedTuple):
    """SPPF's three chained 5x5 max-pools (models/common.py:190-196): channels [0, c) of cat4 [B, h, w, 4c] into
    [c, 2c), [2c, 3c) and [3c, 4c).  Still the tuple ("pool", cat4, h, w, c) for code that unpacks the entry."""
    kind: str
    cat4: torch.Tensor
    h: int
    w: int
    c: int


class TrainEngine:
    def __init__(self, model, B: int, H: int, W: int, device, in_hw=None, arena: Optional[TrainArena] = None,
                 carver: Optional[_Carver] = None, bn_group=None):
        """in_hw: (H_in, W_in) of the input when it differs from the planned (H, W): the plan's first launch is then the
        bilinear resize of train.py's --multi-scale (F.interpolate, align_corners=False) straight into the stem input.
        arena: carve every activation / gradient buffer from that TrainArena (Model.reserve_train_arena); carver: an
        explicit allocator (the arena sizing pass).
        bn_group: a torch.distributed process group: every BatchNorm is a SyncBatchNorm over it (train.py --sync-bn,
        torch.nn.SyncBatchNorm).  Each layer's batch statistics are all-reduced between the stats and finalize launches
        (and its gradient sums in the backward plan), as one fp64 record [sum (C) | sum of squares (C) | pixel count] per
        layer, so ranks may train at different sizes.  With an NCCL group the collectives are captured in the forward
        and backward graphs; with any other backend (gloo) the plans run eagerly."""
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("TrainEngine needs a CUDA device (sm_90a); there is no CPU path")
        det = model.model[-1]
        require_nc(det.nc, "TrainEngine")
        smax = int(max(model.stride))
        if H % smax or W % smax:
            raise RuntimeError(f"image size {H}x{W} must be a multiple of the max stride {smax}")
        self.device, self.B, self.H, self.W = device, B, H, W
        self.in_hw = (H, W) if in_hw is None else (int(in_hw[0]), int(in_hw[1]))
        self.arena = arena
        self._carver = carver if carver is not None else _Carver(arena, device)
        mem0 = torch.cuda.memory_allocated(device)
        self.model = model
        self.layers: List[Union[_BNLayer, _PoolLayer]] = []   # in launch order
        self.pre_ops, self.keep = [], []
        self.flops = 0.0
        L = _lib.lib()
        self._L = L
        mods = list(model.model)
        ch, hw = shapes(mods, H, W)

        def new(h, w, c):
            t = self._carver.take((B, h, w, c), torch.bfloat16)
            self.keep.append(t)
            return t

        out, up_of = route(mods, ch, hw, new)

        def add(mod, x, dst: Slice, res=None, y2x=None, stem=False):
            conv = mod.conv
            k, s, p = ((3, 1), 1, (1, 0)) if stem else (conv.kernel_size[0], conv.stride[0], conv.padding[0])
            z = Slice.full(new(dst.H, dst.W, conv.out_channels))
            lay = _BNLayer(mod, x, z, dst, res, y2x)
            w = conv.weight.detach().float()
            wp, bp = pack_weights(stem_weight(w) if stem else w, None)
            lay.conv = ConvOp(x, wp, bp, w.shape[0], k, s, p, False, out=z)
            lay.wp, lay.stem = wp, stem
            self.flops += lay.conv.info()["flops"]
            self.layers.append(lay)
            return lay

        self.x_s2d = self._carver.take((B, H // 2, W // 2 + 2, 16), torch.bfloat16)
        self._carver.zeroed(self.x_s2d[:, :, 0])    # the pad columns: the stem kernels never write them
        self._carver.zeroed(self.x_s2d[:, :, -1])
        self.sppf = None
        for m in mods:
            i = m.i
            if _is(m, "Detect"):
                break
            fs = sources(m)
            if _is(m, "Conv"):
                if i == 0:
                    add(m, stem_window(self.x_s2d), out[i], stem=True)
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
                self.layers.append(_PoolLayer("pool", cat4, hh, ww, c_))
                add(m.cv2, Slice.full(cat4), out[i])

        # Detect: raw logits per level, fp32 [B, na, H, W, no]
        self.det_out, self.det_convs = [], []
        for l, f in enumerate(det.f):
            mi = det.m[l]
            hh, ww = hw[f]
            if arena is None and carver is None:
                o = torch.empty((B, det.na, hh, ww, det.no), dtype=torch.float32, device=device)
            else:
                o = self._carver.take((B, det.na, hh, ww, det.no), torch.float32)
            wp, bp = pack_weights(mi.weight.detach().float(), mi.bias.detach().float(), MODE_DETECT, det.no)
            stride = float(det.stride[l])
            cv = ConvOp(out[f], wp, bp, mi.weight.shape[0], 1, 1, 0, False,
                        det=dict(out=o, rows_per_image=det.na * hh * ww, row_off=0, no=det.no, decode=False, stride=stride,
                                 anchors_px=(det.anchors[l].detach().float().cpu() * stride).flatten().tolist()))
            self.flops += cv.info()["flops"]
            self.det_out.append(o)
            self.det_convs.append(cv)
        self.out_slices = out
        self.fwd_bytes = self._carver.off   # where the backward plans' buffers start (train_backward.BackwardPlan)
        self.conv_layers = [lay for lay in self.layers if isinstance(lay, _BNLayer)]
        self._bwd, self._pack, self._pack_has_bwd = None, None, False
        self._bwds = {}   # requires_grad flags of model.parameters() -> the BackwardPlan for them; _bwd: the last one run
        self.prof = None  # set to {} to collect per-kernel-kind device times (ms) during forward()
        import os
        self.use_graph = os.environ.get("Y5OBB_NO_GRAPH", "0") != "1"
        self._graphs = {}
        self._nbt = [lay.mod.bn.num_batches_tracked for lay in self.conv_layers]
        self.bn_group = bn_group
        self.bn_rec = None
        if bn_group is not None:
            import torch.distributed as dist
            if dist.get_backend(bn_group) != "nccl":   # (gloo's CUDA all_reduce cannot be captured)
                self.use_graph = False
            # every layer's SyncBatchNorm record [sum | sum of squares | n] in one fp64 buffer, outside the arena
            self.bn_rec = torch.zeros(sum(2 * lay.z.C + 1 for lay in self.conv_layers), dtype=torch.float64, device=device)
            o = 0
            for lay in self.conv_layers:
                lay.rec = self.bn_rec[o:o + 2 * lay.z.C + 1]
                o += 2 * lay.z.C + 1
        cmax = max([lay.z.C for lay in self.conv_layers] + [det.na * 256])
        self.scratch = torch.zeros(int(L.y5obb_bn_scratch_floats(cmax)), dtype=torch.float32, device=device)  # reductions
        # device bytes this plan holds outside the arena (BatchNorm vectors, packed weights, scratch; later the backward
        # plan's and the captured graphs'): with an arena, what each additional training shape costs
        self.outside_bytes = torch.cuda.memory_allocated(device) - mem0

    @property
    def zero_regions(self) -> List[torch.Tensor]:
        """Arena views this plan (forward and backward) relies on being zero: re-zeroed when it runs after another plan."""
        return list(self._carver.zero)

    def _claim_arena(self):
        a = self.arena
        if a is not None and (a.owner is None or a.owner() is not self):
            for t in self._carver.zero:
                t.zero_()
            a.owner = weakref.ref(self)

    _stem_weight = staticmethod(stem_weight)   # layout.stem_weight under the name TrainEngine's callers use

    def refresh_weights(self):
        """Re-pack the (updated) fp32 parameters into the bf16 buffers the TMA descriptors point at — after every
        optimizer.step().  One launch for all layers, forward and data-gradient layouts (csrc/pack_weights.cu)."""
        if self._pack is None:
            from .train_ops import PackPlan, PACK_FWD, PACK_STEM, PACK_DETECT, PACK_DETECT_BIAS
            det = self.model.model[-1]
            ent = []
            for lay in self.conv_layers:
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
        if tuple(x.shape) != (self.B, 3) + self.in_hw:
            raise RuntimeError(f"engine was planned for {(self.B, 3) + self.in_hw}, got {tuple(x.shape)}")
        if x.dtype != torch.uint8:
            x = x.float()
        self._claim_arena()
        if self.prof is not None or not self.use_graph:
            return self._forward_eager(x.contiguous(), refresh)
        slot = self._graphs.setdefault((x.dtype, refresh), dict(calls=0, graph=None, x=None))
        slot["calls"] += 1
        if slot["calls"] == 1:  # first call: eager (warm-up; plans and lazily built state settle)
            return self._forward_eager(x.contiguous(), refresh)
        if slot["graph"] is None:
            if refresh and self._pack is None:
                self.refresh_weights()  # builds the packing plan (allocates): not capturable
            mem0 = torch.cuda.memory_allocated(self.device)
            if self.arena is not None:   # one static input per shape for all plans of the arena
                slot["x"] = self.arena.input_buffer(x.shape, x.dtype)
            else:
                slot["x"] = torch.empty_like(x, memory_format=torch.contiguous_format)
            slot["x"].copy_(x)
            torch.cuda.synchronize(self.device)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, capture_error_mode="thread_local"):
                self._forward_eager(slot["x"], refresh)
            slot["graph"] = g
            self.outside_bytes += torch.cuda.memory_allocated(self.device) - mem0
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
            if self.in_hw != (self.H, self.W):   # --multi-scale: bilinear resize (no flip, no pad) into the stem input
                fn = L.y5obb_scale_img_s2d_u8 if x.dtype == torch.uint8 else L.y5obb_scale_img_s2d
                Hi, Wi = self.in_hw
                run("resize", lambda: fn(x.data_ptr(), self.x_s2d.data_ptr(), self.B, Hi, Wi, self.H, self.W, self.H, self.W,
                                         0, 0.0, 1, st))
            elif x.dtype == torch.uint8:
                run("s2d", lambda: L.y5obb_stem_s2d_u8(x.data_ptr(), self.x_s2d.data_ptr(), self.B, self.H, self.W, 1, st))
            else:
                run("s2d", lambda: L.y5obb_stem_s2d(x.data_ptr(), self.x_s2d.data_ptr(), self.B, self.H, self.W, 1, st))
            for lay in self.layers:
                if isinstance(lay, _PoolLayer):
                    run("pool", lambda: L.y5obb_sppf_pool(lay.cat4.data_ptr(), lay.cat4.shape[3], self.B, lay.h, lay.w, lay.c,
                                                          st))
                    continue
                run("conv", lambda: L.y5obb_conv_run(lay.conv._h, st))
                z, y = lay.z, lay.y
                npix = z.B * z.H * z.W
                bn = lay.mod.bn
                if self.bn_group is None:
                    run("bn_stats", lambda: L.y5obb_bn_batch_stats(
                        z.ptr, z.pix_stride, npix, z.C, bn.weight.data_ptr(), bn.bias.data_ptr(), float(bn.eps),
                        float(bn.momentum), bn.running_mean.data_ptr(), bn.running_var.data_ptr(), lay.scale.data_ptr(),
                        lay.shift.data_ptr(), lay.mean.data_ptr(), lay.invstd.data_ptr(), self.scratch.data_ptr(),
                        self.scratch.numel(), st))
                else:   # SyncBatchNorm: the rank's record, summed over the group, finalised with the global count
                    run("bn_stats", lambda: L.y5obb_bn_stats_sync(z.ptr, z.pix_stride, npix, z.C, lay.rec.data_ptr(),
                                                                  self.scratch.data_ptr(), self.scratch.numel(), st))
                    self._all_reduce(lay.rec)
                    run("bn_finalize", lambda: L.y5obb_bn_finalize_sync(
                        lay.rec.data_ptr(), z.C, bn.weight.data_ptr(), bn.bias.data_ptr(), float(bn.eps), float(bn.momentum),
                        bn.running_mean.data_ptr(), bn.running_var.data_ptr(), lay.scale.data_ptr(), lay.shift.data_ptr(),
                        lay.mean.data_ptr(), lay.invstd.data_ptr(), st))
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

    def _all_reduce(self, rec: torch.Tensor):
        """SUM of a SyncBatchNorm record over bn_group, ordered on the current stream (captured with the graph under NCCL)."""
        import torch.distributed as dist
        dist.all_reduce(rec, op=dist.ReduceOp.SUM, group=self.bn_group)

    def backward(self, grads, trainable=None):
        """grads: dLoss/d(det_out[l]) for the three levels -> the BackwardPlan, whose .flat holds every parameter
        gradient (fp32, model.parameters() order, see train_backward.py).  trainable: requires_grad of every parameter in
        that order (None: the model's current flags).  One plan is kept per set of flags, each with its own graph: frozen
        layers (train.py --freeze) cost no launch, and unfreezing builds the full plan."""
        if trainable is None:
            trainable = [p.requires_grad for p in self.model.parameters()]
        key = tuple(bool(t) for t in trainable)
        plan = self._bwds.get(key)
        if plan is None:
            from .train_backward import BackwardPlan
            mem0 = torch.cuda.memory_allocated(self.device)
            plan = self._bwds[key] = BackwardPlan(self, key)   # packs its data-gradient weights from the current parameters
            self.outside_bytes += torch.cuda.memory_allocated(self.device) - mem0
        elif plan is not self._bwd:
            plan.refresh()                     # its data-gradient weights are as old as its last run
        if plan is not self._bwd:
            self._bwd = plan
            self._pack = None                  # the next refresh_weights() covers its weights too ...
            self._graphs = {}                  # ... so captured forward graphs (old packing plan) are dropped
        plan.run(grads)
        return plan
