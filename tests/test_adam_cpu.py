"""CPU tests of train.py --adam: TrainStep(adam=True)'s parameter groups (train.py:157-163), the host scalars of the fused
Adam step against torch's own expressions, and the refusals of the Adam ABI that happen before any device work."""
import ctypes
import inspect

import numpy as np
import pytest
import torch

from tests.modelgen import build_mirror


def test_adam_parameter_groups():
    from yolov5_obb_b200.train_step import TrainStep, param_groups
    m = build_mirror("n", nc=15, seed=0).train()
    ts = TrainStep(m, batch_size=16, imgsz=1024, ema=False, adam=True)   # on the CPU: no fused step is planned
    opt = ts.optimizer
    assert type(opt) is torch.optim.Adam and not ts._use_fused
    wd = 0.0005 * 16 * 4 / 64                                           # train.py:145 with accumulate = 4
    assert ts.hyp["weight_decay"] == wd
    groups = param_groups(m)
    assert len(opt.param_groups) == 3
    for k, (g, want) in enumerate(zip(opt.param_groups, groups)):
        assert [id(p) for p in g["params"]] == [id(p) for p in want]
        assert g["lr"] == 0.01 and g["betas"] == (0.937, 0.999) and g["eps"] == 1e-8
        assert g["weight_decay"] == (wd if k == 1 else 0.0)
        assert g["foreach"] is True and g["amsgrad"] is False and g["maximize"] is False
        assert not g["capturable"] and not g["fused"] and not g.get("decoupled_weight_decay", False)
        assert "momentum" not in g                                      # the warm-up (train.py:308) leaves betas alone
    sgd = TrainStep(build_mirror("n", nc=15, seed=0).train(), batch_size=16, imgsz=1024, ema=False).optimizer
    assert type(sgd) is torch.optim.SGD and sgd.param_groups[0]["nesterov"] and not ts._fused


def _torch_scalars(lr, beta1, beta2, step):
    """torch/optim/adam.py _multi_tensor_adam, capturable=False, written as there (step is the fp32 CPU state tensor)."""
    from torch.optim.optimizer import _get_value
    bias_correction1 = [1 - beta1 ** _get_value(s) for s in [step]]
    bias_correction2 = [1 - beta2 ** _get_value(s) for s in [step]]
    step_size = [(lr / bc) * -1 for bc in bias_correction1]
    bias_correction2_sqrt = [bc**0.5 for bc in bias_correction2]
    return step_size[0], bias_correction2_sqrt[0]


@pytest.mark.parametrize("betas", [(0.937, 0.999), (0.9, 0.999), (0.3, 0.99)])
def test_host_scalars_equal_torch(betas):
    from yolov5_obb_b200.train_ops import adam_step_scalars
    steps = list(range(1, 50)) + [100, 999, 1000, 1001, 4096, 123457]
    for lr in (0.0, 1e-5, 1e-3, 0.01, 0.0123, 0.1):
        for t in steps:
            st = torch.tensor(float(t), dtype=torch.float32)
            ss, bc2 = adam_step_scalars(lr, betas[0], betas[1], float(t))
            ts, tbc2 = _torch_scalars(lr, betas[0], betas[1], st)
            assert (ss, bc2) == (ts, tbc2), (lr, t)
            assert np.float32(ss) == np.float32(ts) and np.float32(bc2) == np.float32(tbc2)


def test_torch_adam_still_uses_these_expressions():
    """The fused kernel restates this torch's multi-tensor Adam; flag a torch whose expressions moved."""
    from torch.optim import adam
    src = inspect.getsource(adam._multi_tensor_adam)
    for line in ("torch._foreach_lerp_(", "torch._foreach_mul_(device_exp_avg_sqs, beta2)",
                 "step_size = _stack_if_compiling([(lr / bc) * -1 for bc in bias_correction1])",
                 "bias_correction2_sqrt = [bc**0.5 for bc in bias_correction2]",
                 "torch._foreach_div_(exp_avg_sq_sqrt, bias_correction2_sqrt)", "torch._foreach_add_(exp_avg_sq_sqrt, eps)"):
        assert line in src, line


def test_create_refuses_malformed_tables():
    from yolov5_obb_b200 import _lib
    from yolov5_obb_b200.train_ops import AdamEntry
    L = _lib.lib()
    h = ctypes.c_void_p()
    P = 0x1000  # never dereferenced: every table below is refused before any device work
    good = dict(p=P, g=P, exp_avg=P, exp_avg_sq=P, ema=None, n=4, weight_decay=0.0, group=0)
    assert L.y5obb_adam_ema_plan_create(None, 1, ctypes.byref(h)) == 1
    assert L.y5obb_adam_ema_plan_create((AdamEntry * 1)(AdamEntry(**good)), 0, ctypes.byref(h)) == 1
    assert L.y5obb_adam_ema_plan_create((AdamEntry * 1)(AdamEntry(**good)), 1, None) == 1
    for bad in (dict(p=None), dict(g=None), dict(exp_avg=None), dict(exp_avg_sq=None), dict(n=0), dict(n=-1),
                dict(group=3), dict(group=-2), dict(group=-1)):   # group -1 (EMA only) needs an EMA
        arr = (AdamEntry * 2)(AdamEntry(**good), AdamEntry(**{**good, **bad}))
        assert L.y5obb_adam_ema_plan_create(arr, 2, ctypes.byref(h)) == 1, bad
    assert not h.value
    ss = (ctypes.c_float * 3)(-0.01, -0.01, -0.01)
    assert L.y5obb_adam_ema_plan_run(None, ss, 0.9, 0.999, 0.03, 1e-8, 0.0, None) == 1


def test_fused_adam_refuses_mixed_state():
    """Adopting optimizer state needs every parameter's state and one step count."""
    from yolov5_obb_b200.train_ops import FusedAdamEMA
    from yolov5_obb_b200.train_step import param_groups
    m = build_mirror("n", nc=15, seed=0)
    groups = param_groups(m)
    params = [p for g in groups for p in g]
    grads = {p: torch.zeros_like(p) for p in params}
    st = {p: {"step": torch.tensor(3.0), "exp_avg": torch.zeros_like(p), "exp_avg_sq": torch.zeros_like(p)} for p in params}
    partial = dict(list(st.items())[:5])
    with pytest.raises(ValueError, match="all or none"):
        FusedAdamEMA(m, groups, grads, state=partial)
    st[params[7]]["step"] = torch.tensor(2.0)
    with pytest.raises(ValueError, match="step counts differ"):
        FusedAdamEMA(m, groups, grads, state=st)
