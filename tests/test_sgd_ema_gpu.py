"""GPU parity of the fused SGD-Nesterov + EMA step (csrc/sgd_ema.cu) against torch.optim.SGD with the reference's parameter
groups (train.py:148-162) and ModelEMA (utils/torch_utils.py:304-314) over three steps, bit for bit, and of TrainStep's use
of it (tests/test_sgd_exact_gpu.py checks the same at the edges)."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_fused_step_matches_torch_sgd_and_ema():
    from tests.modelgen import build_mirror
    from yolov5_obb_b200.train_ops import FusedSGDEMA
    from yolov5_obb_b200.train_step import ModelEMA, param_groups
    m = build_mirror("n", nc=15, seed=0).to(DEV)
    ref = copy.deepcopy(m)
    lr, mom, wd = (0.01, 0.02, 0.1), 0.937, 5e-4
    g0, g1, g2 = param_groups(ref)
    opt = torch.optim.SGD(g0, lr=lr[0], momentum=mom, nesterov=True)
    opt.add_param_group({"params": g1, "weight_decay": wd, "lr": lr[1]})
    opt.add_param_group({"params": g2, "lr": lr[2]})
    ema_ref = ModelEMA(ref)
    ema = ModelEMA(m)
    grads = {p: torch.zeros_like(p) for p in m.parameters()}
    fused = FusedSGDEMA(m, param_groups(m), grads, ema.ema, weight_decay=wd)
    gen = torch.Generator(device=DEV).manual_seed(0)
    for step in range(3):
        for (p, g), pr in zip(grads.items(), ref.parameters()):
            g.copy_(torch.randn(p.shape, generator=gen, device=DEV))
            pr.grad = g.clone()
        with torch.no_grad():  # BatchNorm running statistics move during training: EMA follows them too
            for b, br in zip(m.buffers(), ref.buffers()):
                if b.dtype.is_floating_point:
                    b.add_(0.01)
                    br.add_(0.01)
        opt.step()
        ema_ref.update(ref)
        ema.updates += 1
        fused.step(lr, mom, ema.decay(ema.updates))
    torch.cuda.synchronize()
    for (n, a), b in zip(m.named_parameters(), ref.parameters()):
        assert torch.equal(a, b), n
        assert torch.equal(fused.mom[a], opt.state[b]["momentum_buffer"]), n
    for (k, a), b in zip(ema.ema.state_dict().items(), ema_ref.ema.state_dict().values()):
        if a.dtype.is_floating_point:
            assert torch.equal(a, b), k


def test_train_step_fused_equals_torch_path():
    """TrainStep with the fused kernel (default) and with torch.optim.SGD + foreach EMA (Y5OBB_FUSED_SGD=0) from the same
    start: after 3 steps on the same batch parameters, momentum buffers and EMA agree to rounding (the two paths consume the
    same device gradients; the backward's split-K atomics make those differ in the last bits between runs)."""
    from tests.modelgen import build_mirror
    from tests.lossgen import synth_targets
    from yolov5_obb_b200.train_step import TrainStep
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    tg = torch.from_numpy(synth_targets(2, 12, 128, nc=15, seed=2)).to(DEV)
    res = []
    for fused in ("1", "0"):
        os.environ["Y5OBB_FUSED_SGD"] = fused
        try:
            m = build_mirror("n", nc=15, seed=0).to(DEV).train()
            ts = TrainStep(m, batch_size=64, imgsz=128)
            assert ts._use_fused == (fused == "1")
            for _ in range(3):
                ts.step(x, tg)
            torch.cuda.synchronize()
            mom = [ts.optimizer.state[p]["momentum_buffer"].clone() for p in m.parameters()]
            res.append(([p.detach().clone() for p in m.parameters()], mom,
                        [v.clone() for v in ts.ema.ema.state_dict().values() if v.dtype.is_floating_point], ts.ema.updates))
        finally:
            os.environ.pop("Y5OBB_FUSED_SGD", None)
    (pa, ma, ea, ua), (pb, mb, eb, ub) = res
    assert ua == ub == 3
    for name, A, B, tol in (("param", pa, pb, 2e-3), ("momentum", ma, mb, 5e-2), ("ema", ea, eb, 2e-3)):
        num = sum(((a - b).double() ** 2).sum().item() for a, b in zip(A, B)) ** 0.5
        den = sum((b.double() ** 2).sum().item() for b in B) ** 0.5
        assert num / den < tol, (name, num / den)
    # the eval plan sees the updated weights (explicit generation counter: the kernel writes through raw pointers)
    m.eval()
    y1, _ = m(x)
    y1 = y1.clone()
    m.invalidate()
    y2, _ = m(x)
    assert torch.equal(y1, y2)
