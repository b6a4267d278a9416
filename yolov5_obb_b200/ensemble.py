"""Model ensembles on the device: models/experimental.py:74-120 (Ensemble, attempt_load), what detect.py and val.py build
for `--weights a.pt b.pt`.

Ensemble.forward(x) is the reference's "nms ensemble": every member runs on the same input (with `augment` passed through,
each member augmenting with its own largest stride) and the members' rows are concatenated along dim 1, in list order;
one NMS then runs over them.  Here the concatenation is never formed: engine.EnsemblePlan stages the image once and each
member's Detect epilogue writes its rows into its own row range of one output (DESIGN.md section 4d).  The Ensemble has the
inference interface of yolo.Model (forward, forward_augment, detect_records, records_plan, tta_plan, stride, names), so
DetectPipeline, Validator and SceneDetector take either."""
import torch
import torch.nn as nn

from .general import DetectRecords


class Ensemble(nn.ModuleList):
    """An eval-mode ensemble of yolo.Model members with one class count, all on one device.  `stride` is the stride tensor of
    the member with the largest max stride (the first such), `names` the last member's (experimental.py:118-119), `nc` the
    common class count.  Plans are cached per (kind, shape, device, slot) and rebuilt when any member's weights changed."""

    def __init__(self, models=()):
        models = list(models)
        if not models:
            raise RuntimeError("an ensemble needs at least one member")
        ncs = [int(m.model[-1].nc) for m in models]
        if len(set(ncs)) != 1:
            raise RuntimeError(f"ensemble members have different class counts {ncs}: their rows cannot be concatenated "
                               "(the reference fails in torch.cat)")
        devs = {next(m.parameters()).device for m in models}
        if len(devs) != 1:
            raise RuntimeError(f"ensemble members are on different devices {sorted(str(d) for d in devs)}")
        if any(m.training for m in models):
            raise RuntimeError("ensemble members must be in eval mode (model.eval()): an ensemble is an inference model")
        super().__init__(models)
        self.training = False
        self.nc = ncs[0]
        self.names = models[-1].names
        self.stride = models[max(range(len(models)), key=lambda i: (float(models[i].stride.max()), -i))].stride
        self._plans = {}

    # ---- nn.Module plumbing
    def train(self, mode: bool = True):
        if mode:
            raise RuntimeError("an ensemble is an inference model: train the members themselves")
        return super().train(False)

    def _apply(self, fn, *args, **kwargs):   # .to() / .cuda(): the plans point at the old storages
        self._plans = {}
        return super()._apply(fn, *args, **kwargs)

    def invalidate(self):
        """Drop every plan; the next call re-plans."""
        self._plans.clear()

    def _precision_key(self):
        """() for the bf16 plans, ("f16",) for the fp16 plans of a half ensemble (engine.plan_dtype)."""
        return self[0]._precision_key()

    def _signature(self):
        return tuple(m._weights_signature() for m in self)

    def _plan(self, kind: str, shape, device, slot: int, compact_detect: bool, augment: bool):
        if self.training or any(m.training for m in self):
            raise RuntimeError("an ensemble is an inference entry point: its members must be in eval mode")
        from .engine import EnsemblePlan
        device = torch.device(device)
        key = (kind, tuple(shape), device.index) + ((int(slot),) if slot else ()) + self._precision_key()
        plan = self._plans.get(key)
        sig = self._signature()
        if plan is None or plan._weights_sig != sig:
            self._plans.pop(key, None)   # (frees the stale plan's buffers before the new one allocates)
            plan = self._plans[key] = EnsemblePlan(list(self), shape[0], shape[2], shape[3], device,
                                                   compact_detect=compact_detect, augment=augment)
            plan._weights_sig = sig
        return plan

    # ---- the inference interface of yolo.Model
    def forward(self, x, augment: bool = False):
        """experimental.py:79-87: (rows [B, sum of the members' rows, nc+185] fp32, None), the members' rows in list order
        (plan-owned buffer, overwritten by the next call).  augment=True: every member's _forward_augment rows."""
        if augment:
            return self.forward_augment(x)
        return self._plan("rows", x.shape, x.device, 0, False, False).forward(x), None

    def forward_augment(self, x):
        """Each member's forward_augment rows (its own gs), member after member: (pred, None)."""
        return self.tta_plan(tuple(x.shape), x.device).forward(x), None

    def tta_plan(self, shape, device, compact_detect: bool = False, slot: int = 0):
        """The engine.EnsemblePlan behind forward_augment / detect_records(augment=True)."""
        return self._plan("tta-records" if compact_detect else "tta", shape, device, slot, compact_detect, True)

    def records_plan(self, shape, device, slot: int = 0):
        """The engine.EnsemblePlan behind detect_records; callers that write its `x_s2d` run it with forward_s2d()."""
        return self._plan("records", shape, device, slot, True, False)

    def detect_records(self, x, slot: int = 0, augment: bool = False):
        """yolo.Model.detect_records over the concatenated rows: a general.DetectRecords for non_max_suppression_obb."""
        if augment:
            plan = self.tta_plan(tuple(x.shape), x.device, compact_detect=True, slot=slot)
        else:
            plan = self.records_plan(tuple(x.shape), x.device, slot)
        return DetectRecords(plan.forward(x), plan.nc, plan.half)


def attempt_load(models):
    """experimental.py:90-120 for models already built (the package has no checkpoint unpickler): a list of eval-mode
    yolo.Model instances -> the model itself for one member, an Ensemble otherwise.  A single model is returned as is."""
    if isinstance(models, nn.Module) and not isinstance(models, nn.ModuleList):
        return models
    models = list(models)
    if len(models) == 1:
        return models[0]
    return Ensemble(models)
