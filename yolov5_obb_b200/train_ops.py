"""ctypes handles for the training-only kernels (BatchNorm backward, layout copies, tensor-core wgrad)."""
import ctypes
from ctypes import c_void_p, c_int, c_int64

import torch

from . import _lib


class WgradDesc(ctypes.Structure):
    """Mirror of y5obb_wgrad_desc (include/y5obb.h)."""
    _fields_ = [("dz", c_void_p), ("dz_pix_stride", c_int64), ("x", c_void_p), ("x_pix_stride", c_int64),
                ("x_row_stride", c_int64), ("x_img_stride", c_int64), ("dw", c_void_p),
                ("dw_tap_stride", c_int64), ("dw_co_stride", c_int64), ("dw_ci_stride", c_int64),
                ("B", c_int), ("Cout", c_int), ("Ho", c_int), ("Wo", c_int), ("Cin", c_int), ("Hi", c_int), ("Wi", c_int),
                ("KH", c_int), ("KW", c_int), ("stride", c_int), ("pad_h", c_int), ("pad_w", c_int),
                ("co_group", c_int), ("co_group_pad", c_int)]


class Wgrad:
    """dW += sum_pixels dz * x over fixed NHWC buffers (TMA descriptors baked at creation).
    dz / x: (ptr, pix_stride) of the channel slice; `keep` holds the owning tensors alive.
    param_layout=False: dw is [KH*KW][Cout][Cin]; True: dw is the nn.Conv2d parameter layout [Cout][Cin][KH][KW].
    co_group=(real, padded): Detect's per-anchor padded channel groups (rows of padding channels are skipped).
    x_strides=(row, image) in elements: explicit strides of x (allows overlapping pixel windows, x_pix_stride < Cin)."""

    def __init__(self, dz_ptr: int, dz_pix_stride: int, x_ptr: int, x_pix_stride: int, dw: torch.Tensor, B, Cout, Ho, Wo,
                 Cin, Hi, Wi, k, stride, pad, keep=(), param_layout=False, co_group=(0, 0), x_strides=(0, 0)):
        kh, kw = (k, k) if isinstance(k, int) else k
        ph, pw = (pad, pad) if isinstance(pad, int) else pad
        st = (1, Cin * kh * kw, kh * kw) if param_layout else (0, 0, 0)
        d = WgradDesc(dz_ptr, dz_pix_stride, x_ptr, x_pix_stride, x_strides[0], x_strides[1], dw.data_ptr(), st[0], st[1], st[2],
                      B, Cout, Ho, Wo, Cin, Hi,
                      Wi, kh, kw, stride, ph, pw, co_group[0], co_group[1])
        rows = Cout if not co_group[1] else Cout // co_group[1] * co_group[0]
        assert dw.dtype == torch.float32 and dw.is_contiguous() and dw.numel() == kh * kw * rows * Cin
        self._keep = (dw,) + tuple(keep)
        self.desc = d  # what the kernel was told (tests/convref.py evaluates it)
        self._h = c_void_p()
        self.device = dw.device
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_wgrad_create(ctypes.byref(d), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_wgrad_create")

    def run(self, stream=None):
        rc = _lib.lib().y5obb_wgrad_run(self._h, stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_wgrad_run")

    SCHEDULE = ("grid", "bk", "kwp", "khp", "T", "ngroups", "BN", "b_chunks", "ci_blks", "co_blks", "a_chunks", "ksplit",
                "steps", "stages")

    def info(self) -> dict:
        """The launch plan the kernel runs (y5obb_wgrad_schedule): grid, pixel block bk = kwp x khp, taps per CTA T and tap
        groups, input-channel block BN (b_chunks chunks, ci_blks blocks), co_blks output-channel blocks of a_chunks chunks,
        split-K factor, pixel blocks `steps` and pipeline stages."""
        v = [c_int() for _ in self.SCHEDULE]
        _lib.check(_lib.lib().y5obb_wgrad_schedule(self._h, *[ctypes.byref(x) for x in v]), "y5obb_wgrad_schedule")
        return {n: x.value for n, x in zip(self.SCHEDULE, v)}

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_wgrad_destroy(h)
            except Exception:
                pass
            self._h = None


PACK_FWD, PACK_DGRAD, PACK_STEM, PACK_DETECT, PACK_DETECT_DGRAD, PACK_DETECT_BIAS, PACK_DGRAD_S2 = range(7)
# PACK_DGRAD with (group_real, group_pad) = (c0, n), n > 0: only the input channels [c0, c0 + n) of the source weight (the data
# gradient of part of a Concat); (0, 0): all of them


class PackEntry(ctypes.Structure):
    """Mirror of y5obb_pack_entry (include/y5obb.h)."""
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("kind", c_int), ("Cout", c_int), ("Cin", c_int), ("KH", c_int),
                ("KW", c_int), ("rows_pad", c_int), ("cols_pad", c_int), ("group_real", c_int), ("group_pad", c_int)]


class PackPlan:
    """All layers' fp32 parameters -> packed bf16 operand buffers in one launch (after every optimiser step).
    entries: (kind, src parameter tensor fp32, dst packed tensor, group_real, group_pad); shapes are read off the tensors
    (PACK_DGRAD: group_real, group_pad = the input-channel window c0, n, or 0, 0 for all)."""

    def __init__(self, entries, device):
        arr = (PackEntry * len(entries))()
        self._keep = []
        for i, (kind, src, dst, g_real, g_pad) in enumerate(entries):
            assert src.dtype == torch.float32 and src.is_contiguous() and dst.is_contiguous()
            if kind == PACK_DETECT_BIAS:
                cout, cin, kh, kw = src.shape[0], 1, 1, 1
                rows_pad, cols_pad = 1, dst.numel()
                assert dst.dtype == torch.float32
            else:
                cout, cin, kh, kw = src.shape
                assert dst.dtype == torch.bfloat16 and dst.dim() == 3
                rows_pad, cols_pad = dst.shape[1], dst.shape[2]
                taps = 3 if kind == PACK_STEM else ((2 if g_real >> 1 else 1) * (2 if g_real & 1 else 1) if kind == PACK_DGRAD_S2 else kh * kw)
                assert dst.shape[0] == taps
            arr[i] = PackEntry(src.data_ptr(), dst.data_ptr(), kind, cout, cin, kh, kw, rows_pad, cols_pad, g_real, g_pad)
            self._keep.append((src, dst))
        self._h = c_void_p()
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_pack_plan_create(arr, len(entries), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_pack_plan_create")

    def run(self, stream=None):
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_pack_plan_run(self._h, stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_pack_plan_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_pack_plan_destroy(h)
            except Exception:
                pass
            self._h = None


class SgdEntry(ctypes.Structure):
    """Mirror of y5obb_sgd_entry (include/y5obb.h)."""
    _fields_ = [("p", c_void_p), ("g", c_void_p), ("mom", c_void_p), ("ema", c_void_p), ("n", c_int64),
                ("weight_decay", ctypes.c_float), ("group", c_int)]


class FusedSGDEMA:
    """optimizer.step() + ema.update() of train.py:336-342 as ONE launch.  Parameters and momentum buffers are bit-equal to
    torch.optim.SGD(nesterov=True)'s foreach step with the reference's parameter groups, and the EMA to ModelEMA's per-tensor
    rule (tests/test_sgd_exact_gpu.py).

    groups: (g0, g1, g2) parameter lists as train.py:148-156 builds them; grads: {parameter: fp32 gradient tensor} with FIXED
    storage (e.g. views of the backward plan's flat buffer); ema_model: a deep copy whose state_dict mirrors model's.
    step(lr=(lr0, lr1, lr2), momentum, ema_decay) applies torch.optim.SGD(nesterov=True) arithmetic and the EMA rule.
    A parameter with requires_grad False (train.py --freeze) is what torch.optim.SGD makes of a parameter without .grad: it
    is not moved and has no momentum buffer; the EMA still follows it.  state: a mapping {parameter: {'momentum_buffer'}}
    such as optimizer.state (after a checkpoint's load_state_dict); its buffers are adopted in place (fp32, contiguous, on
    the parameter's device) and the steps continue from them.  When it holds at least one buffer, a trainable parameter
    without one starts from zeros: round(0 * momentum + g) is torch's clone(grad) up to the sign of a zero."""

    def __init__(self, model, groups, grads, ema_model=None, weight_decay: float = 0.0, state=None):
        self.device = next(model.parameters()).device
        ema_sd = dict(ema_model.state_dict()) if ema_model is not None else {}
        name_of = {id(p): n for n, p in model.named_parameters()}
        self.mom, ent, self._keep = {}, [], []
        adopted = 0
        for gi, plist in enumerate(groups):
            for p in plist:
                e = ema_sd.get(name_of[id(p)])
                if not p.requires_grad:   # frozen: EMA only
                    if e is not None:
                        ent.append(SgdEntry(p.data_ptr(), None, None, e.data_ptr(), p.numel(), 0.0, -1))
                        self._keep += [p, e]
                    continue
                g = grads[p]
                assert p.dtype == torch.float32 and g.dtype == torch.float32 and p.is_contiguous() and g.is_contiguous()
                m = (state.get(p) or {}).get("momentum_buffer") if state is not None else None
                if m is None:
                    m = torch.zeros_like(p)
                else:
                    if m.dtype != torch.float32 or m.device != p.device or m.shape != p.shape or not m.is_contiguous():
                        raise ValueError("FusedSGDEMA: adopted momentum buffers must be contiguous fp32 tensors shaped and "
                                         "placed like their parameter")
                    adopted += 1
                self.mom[p] = m
                ent.append(SgdEntry(p.data_ptr(), g.data_ptr(), m.data_ptr(), e.data_ptr() if e is not None else None, p.numel(),
                                    float(weight_decay) if gi == 1 else 0.0, gi))
                self._keep += [p, g, m, e]
        if ema_model is not None:  # floating-point buffers (BatchNorm running statistics): EMA only
            msd = dict(model.state_dict())
            pnames = set(name_of.values())
            for k, e in ema_sd.items():
                if k in pnames or not e.dtype.is_floating_point:
                    continue
                v = msd[k]
                ent.append(SgdEntry(v.data_ptr(), None, None, e.data_ptr(), v.numel(), 0.0, -1))
                self._keep += [v, e]
        arr = (SgdEntry * len(ent))(*ent)
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_sgd_ema_plan_create(arr, len(ent), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_sgd_ema_plan_create")
        self.steps = 1 if adopted else 0  # adopted buffers already hold a first step

    def step(self, lr, momentum: float, ema_decay: float = 0.0, stream=None):
        lr3 = (ctypes.c_float * 3)(*[float(v) for v in lr])
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_sgd_ema_plan_run(self._h, lr3, float(momentum), float(ema_decay), int(self.steps == 0),
                                                   stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_sgd_ema_plan_run")
        self.steps += 1

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_sgd_ema_plan_destroy(h)
            except Exception:
                pass
            self._h = None


class FusedEMA:
    """ModelEMA.update alone as ONE launch: a table of EMA-only entries (group -1) of the SGD + EMA kernel, one per
    (source, ema) pair of fp32 device tensors with FIXED storage.  step(ema_decay) rounds as the reference's per-tensor
    ops: v *= d; v += (1 - d) * p."""

    def __init__(self, sources, emas):
        ent, self._keep = [], []
        for s, e in zip(sources, emas):
            if s.dtype != torch.float32 or e.dtype != torch.float32 or not s.is_cuda or s.device != e.device or \
                    s.shape != e.shape or not s.is_contiguous() or not e.is_contiguous():
                raise ValueError("FusedEMA: sources and EMA copies must be contiguous fp32 device tensors of one shape")
            ent.append(SgdEntry(s.data_ptr(), None, None, e.data_ptr(), s.numel(), 0.0, -1))
            self._keep += [s, e]
        self.device = self._keep[0].device
        arr = (SgdEntry * len(ent))(*ent)
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_sgd_ema_plan_create(arr, len(ent), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_sgd_ema_plan_create")

    def step(self, ema_decay: float, stream=None):
        lr3 = (ctypes.c_float * 3)(0.0, 0.0, 0.0)
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_sgd_ema_plan_run(self._h, lr3, 0.0, float(ema_decay), 0,
                                                   stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_sgd_ema_plan_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_sgd_ema_plan_destroy(h)
            except Exception:
                pass
            self._h = None


class AdamEntry(ctypes.Structure):
    """Mirror of y5obb_adam_entry (include/y5obb.h)."""
    _fields_ = [("p", c_void_p), ("g", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p), ("ema", c_void_p),
                ("n", c_int64), ("weight_decay", ctypes.c_float), ("group", c_int)]


def adam_step_scalars(lr: float, beta1: float, beta2: float, step: float):
    """(step_size, bias_correction2_sqrt) of torch/optim/adam.py's _multi_tensor_adam (capturable=False) for step count
    `step`, in its fp64 expression order: -lr / (1 - beta1^t) and (1 - beta2^t)^0.5.  The kernel reads both as fp32, as
    ATen's foreach kernels read the Python floats."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    return (lr / bias_correction1) * -1, bias_correction2 ** 0.5


class FusedAdamEMA:
    """optimizer.step() of torch.optim.Adam (train.py --adam, train.py:157-163: coupled L2 weight decay, amsgrad off) +
    ema.update() as ONE launch.  Parameters, exp_avg and exp_avg_sq are bit-equal to torch's foreach step, and the EMA to
    ModelEMA's per-tensor rule (tests/test_adam_ema_gpu.py).

    groups, grads, ema_model, weight_decay: as FusedSGDEMA (weight decay on group 1 only).  state: a mapping
    {parameter: {'step', 'exp_avg', 'exp_avg_sq'}} such as optimizer.state; where it holds every parameter the moments are
    adopted in place (fp32, contiguous, on the parameter's device) and the step count is theirs, which must be one count for
    all.  `self.state` is torch.optim.Adam's per-parameter state: the moments the kernel updates and a 'step' that is a view
    of one CPU fp32 tensor, `step_count`, advanced by one op per step.  step(lr=(lr0, lr1, lr2), betas, eps, ema_decay).
    A parameter with requires_grad False (train.py --freeze) is not moved and has no state, as torch.optim.Adam treats a
    parameter without .grad; the EMA still follows it.  "All or none" and the one step count apply to the trainable ones."""

    def __init__(self, model, groups, grads, ema_model=None, weight_decay: float = 0.0, state=None):
        self.device = next(model.parameters()).device
        ema_sd = dict(ema_model.state_dict()) if ema_model is not None else {}
        name_of = {id(p): n for n, p in model.named_parameters()}
        params = [p for plist in groups for p in plist if p.requires_grad]
        adopted = [state.get(p) if state is not None else None for p in params]
        n_have = sum(1 for s in adopted if s)
        if n_have not in (0, len(params)):
            raise ValueError(f"FusedAdamEMA: optimizer state holds {n_have} of {len(params)} parameters; it adopts all or none")
        steps = {float(s["step"]) for s in adopted if s}
        if len(steps) > 1:
            raise ValueError(f"FusedAdamEMA: the parameters' Adam step counts differ ({sorted(steps)}); the fused step needs one")
        self.t = steps.pop() if steps else 0.0
        self.step_count = torch.full((len(params),), self.t, dtype=torch.float32)
        self.state, ent, self._keep = {}, [], []
        i = 0
        for gi, plist in enumerate(groups):
            for p in plist:
                if not p.requires_grad:   # frozen: EMA only
                    e = ema_sd.get(name_of[id(p)])
                    if e is not None:
                        ent.append(AdamEntry(p.data_ptr(), None, None, None, e.data_ptr(), p.numel(), 0.0, -1))
                        self._keep += [p, e]
                    continue
                g = grads[p]
                assert p.dtype == torch.float32 and g.dtype == torch.float32 and p.is_contiguous() and g.is_contiguous()
                s = adopted[i]
                if s:
                    m, v = s["exp_avg"], s["exp_avg_sq"]
                    for t in (m, v):
                        if t.dtype != torch.float32 or t.device != p.device or t.shape != p.shape or not t.is_contiguous():
                            raise ValueError("FusedAdamEMA: adopted moments must be contiguous fp32 tensors shaped and placed "
                                             "like their parameter")
                else:
                    m, v = torch.zeros_like(p), torch.zeros_like(p)
                self.state[p] = {"step": self.step_count[i], "exp_avg": m, "exp_avg_sq": v}
                e = ema_sd.get(name_of[id(p)])
                ent.append(AdamEntry(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(),
                                     e.data_ptr() if e is not None else None, p.numel(),
                                     float(weight_decay) if gi == 1 else 0.0, gi))
                self._keep += [p, g, m, v, e]
                i += 1
        if ema_model is not None:  # floating-point buffers (BatchNorm running statistics): EMA only
            msd = dict(model.state_dict())
            pnames = set(name_of.values())
            for k, e in ema_sd.items():
                if k in pnames or not e.dtype.is_floating_point:
                    continue
                b = msd[k]
                ent.append(AdamEntry(b.data_ptr(), None, None, None, e.data_ptr(), b.numel(), 0.0, -1))
                self._keep += [b, e]
        arr = (AdamEntry * len(ent))(*ent)
        self._h = c_void_p()
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_adam_ema_plan_create(arr, len(ent), ctypes.byref(self._h))
        _lib.check(rc, "y5obb_adam_ema_plan_create")

    def step(self, lr, betas, eps: float, ema_decay: float = 0.0, stream=None):
        t = self.t + 1.0          # torch advances `step` before it forms the bias corrections
        b1, b2 = float(betas[0]), float(betas[1])
        scal = [adam_step_scalars(float(v), b1, b2, t) for v in lr]
        ss = (ctypes.c_float * 3)(*[s for s, _ in scal])
        with torch.cuda.device(self.device):
            rc = _lib.lib().y5obb_adam_ema_plan_run(self._h, ss, b1, b2, scal[0][1], float(eps), float(ema_decay),
                                                    stream if stream is not None else _lib.stream_ptr(self.device))
        _lib.check(rc, "y5obb_adam_ema_plan_run")
        self.step_count.add_(1)   # every parameter's state['step'] at once
        self.t = t

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().y5obb_adam_ema_plan_destroy(h)
            except Exception:
                pass
            self._h = None
