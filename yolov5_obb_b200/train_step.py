"""One optimisation step of train.py:296-342 (the loop body), driven through the same entry points:

    pred = model(imgs)                       # models/yolo.py Model.forward   -> train_engine / train_backward kernels
    loss, items = compute_loss(pred, tgts)   # utils/loss.py ComputeLoss      -> csrc/loss.cu
    loss.backward()                          # train.py:333
    [one all-reduce of the flat gradient]    # DDP's gradient averaging of a loss x WORLD_SIZE (train.py:328) == a SUM over ranks
    optimizer.step(); optimizer.zero_grad(); ema.update(model)   # train.py:336-342

Parameter groups follow train.py:148-162 (BatchNorm weights: no decay; other weights: weight decay; biases),
SGD with Nesterov momentum (train.py:158) or, with adam=True, Adam (train.py --adam, train.py:157-163),
ModelEMA as utils/torch_utils.py:284-314.
The device computes in bf16 with fp32 accumulation and fp32 master weights: no loss scaling is needed (the reference's
GradScaler exists for fp16 autocast, train.py:246,333-337)."""
import math
import random
from copy import deepcopy
from typing import Optional

import torch
import torch.distributed as dist
import torch.nn as nn

from .loss import ComputeLoss

# data/hyps/obb/hyp.finetune_dota.yaml (the reference's shipped hyper-parameters for DOTA)
HYP_FINETUNE_DOTA = dict(lr0=0.01, lrf=0.2, momentum=0.937, weight_decay=0.0005, warmup_epochs=3.0, warmup_momentum=0.8,
                         warmup_bias_lr=0.1, box=0.05, cls=0.5, cls_pw=1.0, theta=0.5, theta_pw=1.0, obj=1.0, obj_pw=1.0,
                         iou_t=0.2, anchor_t=4.0, fl_gamma=0.0, cls_theta=180, csl_radius=2.0)


def param_groups(model):
    """train.py:148-156: g0 = BatchNorm weights (no decay), g1 = other weights (decay), g2 = biases."""
    g0, g1, g2 = [], [], []
    for v in model.modules():
        if hasattr(v, "bias") and isinstance(v.bias, nn.Parameter):
            g2.append(v.bias)
        if isinstance(v, nn.BatchNorm2d):
            g0.append(v.weight)
        elif hasattr(v, "weight") and isinstance(v.weight, nn.Parameter):
            g1.append(v.weight)
    return g0, g1, g2


def freeze_layers(model, freeze=(0,)):
    """train.py:126-131 (--freeze): [n] freezes layers 0..n-1, a longer list exactly the layers it names.  A parameter whose
    name contains f"model.{x}." for a frozen x gets requires_grad False, every other one True.  Returns the frozen names."""
    freeze = [f"model.{x}." for x in (freeze if len(freeze) > 1 else range(freeze[0]))]
    frozen = []
    for k, v in model.named_parameters():
        v.requires_grad = True
        if any(x in k for x in freeze):
            v.requires_grad = False
            frozen.append(k)
    return frozen


def multi_scale_shape(imgsz: int, gs: int, H: int, W: int, rng: random.Random):
    """train.py:314-318 (--multi-scale) for a batch of H x W images: one draw from `rng` -> (ns_h, ns_w, label_ratio).
    The reference passes float bounds to randrange, which Python 3.12 refuses; their integral values give the draws Python
    3.8-3.11 gave."""
    sz = rng.randrange(int(imgsz * 0.5), int(imgsz * 1.5 + gs)) // gs * gs
    return _scaled_shape(sz, gs, H, W)


def _scaled_shape(sz: int, gs: int, H: int, W: int):
    """sf == 1 leaves the batch alone: (H, W, 1.0).  The fp64 ceil is kept as written: for some sizes it rounds up one grid
    step (imgsz 800, sz 448 -> 480)."""
    sf = sz / max(H, W)
    if sf == 1:
        return H, W, 1.0
    ns = [math.ceil(x * sf / gs) * gs for x in (H, W)]
    return ns[0], ns[1], float(ns[0]) / H


def multi_scale_max_shape(imgsz: int, gs: int, H: int, W: int):
    """The largest (ns_h, ns_w) multi_scale_shape can return for H x W batches."""
    shapes = [_scaled_shape(v // gs * gs, gs, H, W) for v in range(int(imgsz * 0.5), int(imgsz * 1.5 + gs))]
    return max(s[0] for s in shapes), max(s[1] for s in shapes)


class ModelEMA:
    """utils/torch_utils.py:284-314: EMA of every floating-point state_dict entry, decay ramp d*(1-exp(-n/2000)).
    update() rounds as the reference's per-tensor `v *= d; v += (1 - d) * msd[k]` does: the product (1 - d) * p is rounded
    before the add (an alpha add would fuse it into one FMA).  On the device, with fp32 entries, it is one launch of the
    SGD + EMA kernel over an EMA-only table (train_ops.FusedEMA); elsewhere the same rule as foreach ops."""

    def __init__(self, model, decay=0.9999, updates=0):
        engines = getattr(model, "_engines", None)
        if engines is not None:  # plans hold device handles: never copied
            model._engines = {}
        self.ema = deepcopy(model).eval()
        if engines is not None:
            model._engines = engines
        self.updates = updates
        self.decay = lambda x: decay * (1 - math.exp(-x / 2000))
        for p in self.ema.parameters():
            p.requires_grad_(False)
        self._pairs = None
        self._fused = None

    def update(self, model):
        with torch.no_grad():
            self.updates += 1
            d = self.decay(self.updates)
            if self._pairs is None:
                msd = model.state_dict()
                ev, mv = [], []
                for k, v in self.ema.state_dict().items():
                    if v.dtype.is_floating_point:
                        ev.append(v)
                        mv.append(msd[k].detach())
                self._pairs = (ev, mv)
                if ev and all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in ev + mv):
                    from .train_ops import FusedEMA
                    self._fused = FusedEMA(mv, ev)
            if self._fused is not None:
                self._fused.step(d)
                if hasattr(self.ema, "_bump_generation"):
                    self.ema._bump_generation()   # written through raw pointers: inference plans must re-fold the EMA
                return
            ev, mv = self._pairs
            torch._foreach_mul_(ev, d)
            torch._foreach_add_(ev, torch._foreach_mul(mv, 1 - d))


class TrainStep:
    """model: yolov5_obb_b200.yolo.Model on a CUDA device, in train() mode.  step(imgs, targets) -> (loss, loss_items)."""

    def __init__(self, model, hyp: Optional[dict] = None, batch_size: int = 16, imgsz: int = 1024, ema: bool = True,
                 warmup_iters: int = 0, multi_scale: bool = False, seed: Optional[int] = None, adam: bool = False,
                 freeze=(0,), sync_bn: bool = False):
        """warmup_iters > 0: the warm-up of train.py:305-316 over that many iterations (the reference uses
        max(round(warmup_epochs * batches_per_epoch), 1000)): every group's lr is interpolated from 0 (biases: from
        hyp['warmup_bias_lr']) to lr0 and the momentum from hyp['warmup_momentum'] to hyp['momentum'].

        multi_scale=True: train.py --multi-scale (train.py:312-320).  Every step draws a size (multi_scale_shape), resizes
        the batch on the device as the plan's first launch and scales targets[:, 2:6] into a buffer the step owns (the
        caller's targets are left as they are; the reference scales them in place).  The draws come from a
        random.Random(seed) owned by the step, seed=None meaning train.py's init_seeds(1 + RANK): the module-level
        `random` stays the augmentation's (augment.DeviceAugmentLoader), as in the reference with dataloader workers,
        where the main process draws nothing else from it.  The constructor reserves one training arena
        (Model.reserve_train_arena) for batch_size images of the largest drawable size, assuming imgsz x imgsz batches
        (no --rect), so an out-of-memory error shows at start-up.  `last_shape` is the (h, w) the last step trained at.

        adam=True: train.py --adam.  The optimizer is torch.optim.Adam(g0, lr=lr0, betas=(momentum, 0.999)) with g1 (weight
        decay) and g2 added as for SGD; Adam groups have no 'momentum', so the warm-up moves only the learning rates.  The
        fused step (below) keeps torch's own per-parameter state in optimizer.state, so optimizer.state_dict() is the
        reference's checkpoint format, and after optimizer.load_state_dict() the next step continues from the loaded
        moments and step count.

        freeze: train.py --freeze, applied by freeze_layers before the optimizer and the EMA are built ([10]: the backbone,
        [0, 1, 2]: those layers; [0]: nothing).  Frozen parameters stay in their parameter groups; the optimizer leaves them
        as they are and keeps no state for them, the EMA follows them, and the backward plan computes no gradient that
        only they would need.  requires_grad may also be changed between steps (unfreezing after some epochs): the next
        step builds the plan for the new flags.  With adam=True, once a frozen parameter becomes trainable torch.optim.Adam
        keeps a step count per parameter, which the fused kernel cannot follow: the step then uses torch.optim.Adam and
        the foreach EMA for the rest of the run.

        sync_bn=True: train.py --sync-bn (torch.nn.SyncBatchNorm.convert_sync_batchnorm, train.py:207-210).  In an
        initialised process group of more than one rank, every BatchNorm of the training plans uses the batch statistics
        of all ranks (the default group: model.bn_group), its per-layer sums and pixel counts all-reduced inside the
        forward plan and its gradient sums inside the backward plan; running statistics come out identical on every rank.
        Otherwise (no group, or one rank) the plans are the plain ones, as SyncBatchNorm falls back to batch_norm."""
        self.model = model
        self.hyp = dict(HYP_FINETUNE_DOTA if hyp is None else hyp)
        nbs = 64
        self.accumulate = max(round(nbs / batch_size), 1)
        self.hyp["weight_decay"] *= batch_size * self.accumulate / nbs  # train.py:145
        nl = model.model[-1].nl
        self.hyp["box"] *= 3.0 / nl                                     # train.py:249-252
        self.hyp["cls"] *= model.model[-1].nc / 80.0 * 3.0 / nl
        self.hyp["obj"] *= (imgsz / 640) ** 2 * 3.0 / nl
        self.hyp["theta"] *= 3.0 / nl
        self.hyp["label_smoothing"] = 0.0
        model.hyp = self.hyp
        model.nc = model.model[-1].nc
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        rank = dist.get_rank() if self.world > 1 else -1
        self.multi_scale, self.imgsz = bool(multi_scale), int(imgsz)
        self.gs = max(int(model.stride.max()), 32)                     # train.py:134
        self.rng = random.Random(1 + rank if seed is None else seed)
        self.last_shape = None
        self._tg = None
        if self.world > 1:
            # DDP broadcasts rank 0's parameters and buffers when it wraps the model (train.py:214); the reference seeds
            # per rank (train.py:100), so without this the replicas would start from different weights.  Done BEFORE the
            # optimizer and the EMA copy are built.
            from .dist_util import broadcast_model_state
            broadcast_model_state(model, 0)
            if hasattr(model, "_bump_generation"):
                model._bump_generation()
        self.sync_bn = bool(sync_bn) and self.world > 1
        model.bn_group = dist.group.WORLD if self.sync_bn else None
        freeze_layers(model, freeze)
        if not any(p.requires_grad for p in model.parameters()):
            raise RuntimeError(f"freeze={list(freeze)} freezes every parameter of the model: nothing is left to train")
        g0, g1, g2 = param_groups(model)
        self.adam = bool(adam)
        if self.adam:
            self.optimizer = torch.optim.Adam(g0, lr=self.hyp["lr0"], betas=(self.hyp["momentum"], 0.999), foreach=True)
        else:
            self.optimizer = torch.optim.SGD(g0, lr=self.hyp["lr0"], momentum=self.hyp["momentum"], nesterov=True,
                                             foreach=True)
        self.optimizer.add_param_group({"params": g1, "weight_decay": self.hyp["weight_decay"]})
        self.optimizer.add_param_group({"params": g2})
        self.ema = ModelEMA(model) if ema else None
        self.compute_loss = ComputeLoss(model)
        self.ni = 0
        self.warmup_iters = int(warmup_iters)
        self._last_opt = -1
        self.optimizer.zero_grad(set_to_none=True)
        # optimizer.step() + ema.update() as ONE kernel (csrc/sgd_ema.cu, SURVEY 8f rank 1) whenever every batch ends with an
        # optimizer step (accumulate == 1: the gradient of the step is exactly the backward plan's flat buffer).  With gradient
        # accumulation torch.optim.SGD / Adam + ModelEMA.update stay in charge.  Y5OBB_FUSED_SGD=0 forces the torch path for
        # either optimizer.
        import os
        self._fused = None
        self._fused_state = None
        self._fused_flags = None
        self._use_fused = (self.accumulate == 1 and os.environ.get("Y5OBB_FUSED_SGD", "1") != "0"
                           and next(model.parameters()).is_cuda and hasattr(model, "_bump_generation"))
        if self.multi_scale:
            hmax, wmax = multi_scale_max_shape(self.imgsz, self.gs, self.imgsz, self.imgsz)
            model.reserve_train_arena(batch_size, hmax, wmax, next(model.parameters()).device)

    def step(self, imgs: torch.Tensor, targets: torch.Tensor):
        """imgs: uint8 or float [B,3,H,W] on the device; targets [nt, 187] (image index, class, cx, cy, l, s, theta, CSL row)."""
        model = self.model
        if self.ni <= self.warmup_iters and self.warmup_iters > 0:   # train.py:305-316 (np.interp on [0, nw]; lf(epoch 0) = 1)
            f = self.ni / self.warmup_iters
            for j, g in enumerate(self.optimizer.param_groups):
                lo = self.hyp["warmup_bias_lr"] if j == 2 else 0.0
                g["lr"] = lo + f * (self.hyp["lr0"] - lo)
                if "momentum" in g:
                    g["momentum"] = self.hyp["warmup_momentum"] + f * (self.hyp["momentum"] - self.hyp["warmup_momentum"])
        size = None
        if self.multi_scale:                                # train.py:312-320
            H, W = int(imgs.shape[2]), int(imgs.shape[3])
            nh, nw, ratio = multi_scale_shape(self.imgsz, self.gs, H, W, self.rng)
            if (nh, nw) != (H, W):
                size = (nh, nw)
                targets = self._scale_targets(targets, ratio)
            self.last_shape = (nh, nw)
            pred = model.forward_train(imgs, size)          # the resize is the plan's first launch
        else:
            self.last_shape = (int(imgs.shape[2]), int(imgs.shape[3]))
            pred = model(imgs)                              # uint8 is normalised inside the stem's loader kernel
        loss, items = self.compute_loss(pred, targets)
        loss.backward()                                     # (x WORLD_SIZE of train.py:328 is folded into the SUM below)
        if self.ni - self._last_opt >= self.accumulate:
            if self._use_fused and self.adam and self._unfrozen():
                self._leave_fused_adam()
            if self._use_fused:
                self._fused_step()
            else:
                if self.world > 1:
                    self._allreduce_grads()
                self.optimizer.step()
                self.optimizer.zero_grad(set_to_none=True)
                if self.ema is not None:
                    self.ema.update(model)
            self._last_opt = self.ni
        self.ni += 1
        return loss.detach(), items

    def _scale_targets(self, targets: torch.Tensor, ratio: float) -> torch.Tensor:
        """targets[:, 2:6] * label_ratio (cx, cy, l, s in the 187-, 8- and 7-column layouts; fp32 as ATen's in-place
        multiply computes it) in a buffer the step owns, reused (stream-ordered) by later steps."""
        nt = int(targets.shape[0])
        t = self._tg
        if t is None or t.shape[0] < nt or t.shape[1:] != targets.shape[1:] or t.dtype != targets.dtype or \
                t.device != targets.device:
            t = self._tg = torch.empty((max(nt, 64) * 2,) + tuple(targets.shape[1:]), dtype=targets.dtype,
                                       device=targets.device)
        out = t[:nt]
        out.copy_(targets)
        out[:, 2:6].mul_(ratio)
        return out

    def run(self, host_batches):
        """The batch loop of train.py:296-342 over HOST batches (what the dataloader yields: pinned uint8 images [B,3,H,W] and
        float targets [nt, 187 | 8 | 7]): yields (loss, loss_items) per batch, in order, as HOST tensors.
        `imgs.to(device, non_blocking=True)` of train.py:300 becomes a copy of batch i+1 on a second stream while step i
        computes (two device buffers per input, event-ordered), and the loss of step i - the one device->host read the loop
        needs (train.py:344-348 mloss) - is fetched after step i+1 has been queued, so the compute stream never drains."""
        dev = next(self.model.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("TrainStep.run needs the model on a CUDA device; there is no CPU path")
        main = torch.cuda.current_stream(dev)
        io = getattr(self, "_io", None)
        if io is None:
            ev = torch.cuda.Event
            io = self._io = dict(copy=torch.cuda.Stream(dev), img=[None, None], tg=[None, None], copied=[ev(), ev()],
                                 consumed=[ev(), ev()], host=[None, None], done=[ev(), ev()])
        copy = io["copy"]

        def upload(j, batch, wait):
            imgs_h, tg_h = batch
            nt = int(tg_h.shape[0])
            if io["img"][j] is None or io["img"][j].shape != imgs_h.shape or io["img"][j].dtype != imgs_h.dtype:
                if wait:
                    io["consumed"][j].synchronize()
                    wait = False
                io["img"][j] = torch.empty(imgs_h.shape, dtype=imgs_h.dtype, device=dev)
            t = io["tg"][j]
            if t is None or t.shape[0] < nt or t.shape[1:] != tg_h.shape[1:] or t.dtype != tg_h.dtype:
                if wait:
                    io["consumed"][j].synchronize()
                    wait = False
                io["tg"][j] = torch.empty((max(nt, 64) * 2,) + tuple(tg_h.shape[1:]), dtype=tg_h.dtype, device=dev)
            with torch.cuda.stream(copy):
                if wait:
                    copy.wait_event(io["consumed"][j])      # the step that used these buffers has been through them
                io["img"][j].copy_(imgs_h, non_blocking=True)
                if nt:
                    io["tg"][j][:nt].copy_(tg_h, non_blocking=True)
                io["copied"][j].record(copy)
            return nt

        def finish(p):
            h, e = p
            e.synchronize()
            return h[0].clone(), h[1:].clone()

        it = iter(host_batches)
        cur = next(it, None)
        if cur is None:
            return
        for e in io["consumed"]:       # a previous run() that was abandoned half-way may still own the buffers
            e.synchronize()
        copy.wait_stream(main)
        used = [False, False]
        nt = upload(0, cur, False)
        used[0] = True
        i, pending = 0, None
        while cur is not None:
            j = i & 1
            nxt = next(it, None)
            nt_next = 0
            if nxt is not None:
                nt_next = upload(j ^ 1, nxt, used[j ^ 1])
                used[j ^ 1] = True
            main.wait_event(io["copied"][j])
            loss, items = self.step(io["img"][j], io["tg"][j][:nt])
            io["consumed"][j].record(main)
            if io["host"][j] is None or io["host"][j].numel() != 1 + items.numel():
                io["host"][j] = torch.empty(1 + items.numel(), dtype=torch.float32).pin_memory()
            io["host"][j].copy_(torch.cat([loss.detach().reshape(1).float(), items.detach().reshape(-1).float()]), non_blocking=True)
            io["done"][j].record(main)
            if pending is not None:
                yield finish(pending)
            pending = (io["host"][j], io["done"][j])
            cur, nt = nxt, nt_next
            i += 1
        if pending is not None:
            yield finish(pending)

    def _unfrozen(self) -> bool:
        """Whether the last backward trained a parameter that the fused table holds as frozen."""
        flags = self.model._last_train_engine._bwd.trainable
        return self._fused is not None and any(t and not f for t, f in zip(flags, self._fused_flags))

    def _leave_fused_adam(self):
        """torch.optim.Adam + the foreach EMA from this step on: each parameter's state gets its own step count."""
        for st in self.optimizer.state.values():
            if "step" in st:
                st["step"] = st["step"].clone()
        self._use_fused, self._fused = False, None

    def _fused_step(self):
        """train.py:336-342 (optimizer.step, zero_grad, ema.update) as one launch over a device-resident tensor table.
        Gradients are read in place from the backward plan's flat fp32 buffer (all-reduced in place first when N > 1);
        learning rates / momentum are taken from optimizer.param_groups every step, so warm-up schedules that edit them
        (train.py:305-316) keep working; the momentum buffers are registered in optimizer.state for checkpoints.
        Adam: lr, betas and eps are read the same way, and optimizer.state holds torch's exp_avg / exp_avg_sq / step, which
        the kernel updates in place.  optimizer.load_state_dict() replaces optimizer.state, so for either optimizer a new
        state object means a checkpoint was loaded: the table is rebuilt on the loaded tensors."""
        from .train_ops import FusedAdamEMA, FusedSGDEMA
        model = self.model
        plan = model._last_train_engine._bwd
        if self.world > 1:
            dist.all_reduce(plan.flat, op=dist.ReduceOp.SUM)
        key = plan.flat if plan.arena is not None else plan   # (an arena's flat buffer is shared by every shape)
        ema = self.ema.ema if self.ema is not None else None
        opt = self.optimizer
        # (re)built for the plan's buffer and for its trainable flags: frozen parameters are EMA-only entries
        rebuild = self._fused is None or self._fused_plan is not key or self._fused_flags != plan.trainable
        if self.adam:
            if rebuild or self._fused_state is not opt.state:
                groups = [g["params"] for g in opt.param_groups]
                self._fused = FusedAdamEMA(model, groups, plan.pgrad, ema, weight_decay=self.hyp["weight_decay"],
                                           state=opt.state)
                self._fused_plan, self._fused_flags = key, plan.trainable
                for p, s in self._fused.state.items():
                    opt.state[p] = s
                self._fused_state = opt.state
        elif rebuild or self._fused_state is not opt.state:
            groups = [g["params"] for g in opt.param_groups]
            # adopts the buffers optimizer.state holds: a loaded checkpoint's, or this run's (the buffers of parameters frozen
            # since stay there, and torch's SGD resumes from them after an unfreeze)
            self._fused = FusedSGDEMA(model, groups, plan.pgrad, ema, weight_decay=self.hyp["weight_decay"], state=opt.state)
            self._fused_plan, self._fused_flags = key, plan.trainable
            for p, m in self._fused.mom.items():
                opt.state[p]["momentum_buffer"] = m
            self._fused_state = opt.state
        g = opt.param_groups
        if self.adam:
            betas, eps = g[0]["betas"], g[0]["eps"]
            if any(tuple(x["betas"]) != tuple(betas) or x["eps"] != eps for x in g[1:]):
                raise ValueError("the fused Adam step needs one (betas, eps) for every parameter group; "
                                 "set Y5OBB_FUSED_SGD=0 to step per group with torch.optim.Adam")
        elif any(x["momentum"] != g[0]["momentum"] for x in g[1:]):
            raise ValueError("the fused SGD step needs one momentum for every parameter group; "
                             "set Y5OBB_FUSED_SGD=0 to step per group with torch.optim.SGD")
        d = 0.0
        if self.ema is not None:
            self.ema.updates += 1
            d = self.ema.decay(self.ema.updates)
        if self.adam:
            self._fused.step((g[0]["lr"], g[1]["lr"], g[2]["lr"]), betas, eps, d)
        else:
            self._fused.step((g[0]["lr"], g[1]["lr"], g[2]["lr"]), g[0]["momentum"], d)
        self.optimizer.zero_grad(set_to_none=True)
        model._bump_generation()   # parameters changed through raw pointers: inference plans must re-fold them
        if self.ema is not None and hasattr(self.ema.ema, "_bump_generation"):
            self.ema.ema._bump_generation()

    def _allreduce_grads(self):
        """DDP averages the gradients of a loss that train.py:328 multiplied by WORLD_SIZE: the net effect is the SUM
        of the per-rank gradients.  The parameter gradients are views of one flat buffer (yolo._TrainFn.backward),
        so this is ONE NCCL all-reduce over NVLink; gradients that are not (accumulation into pre-existing .grad
        tensors) are reduced one by one."""
        params = [p for p in self.model.parameters() if p.grad is not None]
        eng = getattr(self.model, "_last_train_engine", None)
        if getattr(eng, "arena", None) is not None:
            eng = eng.arena
        cands = [getattr(eng, "last_grad_flat", None)]
        if params and params[0].grad._base is not None:   # gradient accumulation: .grad still views the FIRST step's buffer
            cands.append(params[0].grad._base)
        for flat in cands:
            if flat is None or flat.dim() != 1:
                continue
            lo, hi = flat.data_ptr(), flat.data_ptr() + flat.numel() * flat.element_size()
            if all(lo <= p.grad.data_ptr() and p.grad.data_ptr() + p.grad.numel() * p.grad.element_size() <= hi for p in params):
                dist.all_reduce(flat, op=dist.ReduceOp.SUM)
                return
        for p in params:
            dist.all_reduce(p.grad, op=dist.ReduceOp.SUM)
