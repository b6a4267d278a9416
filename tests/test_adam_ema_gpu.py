"""GPU parity of the fused Adam + EMA step (csrc/sgd_ema.cu k_adam_ema, train_ops.FusedAdamEMA) against torch.optim.Adam's
foreach step with the reference's parameter groups (train.py --adam, train.py:157-163) and ModelEMA, and of TrainStep(adam=True):
fused against torch path, checkpoint / resume through optimizer.state_dict(), gradient accumulation, ABI refusals."""
import copy
import ctypes
import gc
import io
import os

import pytest
import torch

from tests.lossgen import synth_targets
from tests.modelgen import build_mirror

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WD = 5e-4


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """Models, plans and optimizer state of these tests are freed, and their cached blocks returned to the device, before
    the next module: later modules (whole-scene detection) allocate single buffers of tens of GB."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _lrs(step):
    """Per-group learning rates that change every step; step 0 is the warm-up's first: weights at 0, biases at 0.1."""
    return (0.0, 0.0, 0.1) if step == 0 else (0.002 * step, 0.003 * step, 0.1 - 0.02 * step)


def _grad(shape, gen):
    """Seeded gradients over six decades, with about 10 % exact zeros and 10 % values near 1e-30."""
    g = torch.randn(shape, generator=gen, device=DEV)
    g = g * 10.0 ** (torch.rand(shape, generator=gen, device=DEV) * 6 - 4)
    u = torch.rand(shape, generator=gen, device=DEV)
    g = torch.where(u < 0.1, torch.zeros_like(g), g)
    return torch.where((u >= 0.1) & (u < 0.2), torch.randn(shape, generator=gen, device=DEV) * 1e-30, g)


def _torch_adam(model, betas):
    from yolov5_obb_b200.train_step import param_groups
    g0, g1, g2 = param_groups(model)
    opt = torch.optim.Adam(g0, lr=0.01, betas=betas, foreach=True)
    opt.add_param_group({"params": g1, "weight_decay": WD})
    opt.add_param_group({"params": g2})
    return opt


def _fused(model, grads, ema=None, state=None):
    from yolov5_obb_b200.train_ops import FusedAdamEMA
    from yolov5_obb_b200.train_step import param_groups
    return FusedAdamEMA(model, param_groups(model), grads, ema, weight_decay=WD, state=state)


@pytest.mark.parametrize("betas", [(0.937, 0.999), (0.3, 0.99)])   # lerp weight below / above 0.5: ATen's two lerp forms
def test_fused_adam_bit_equal_to_torch_adam_and_ema(betas):
    from yolov5_obb_b200.train_step import ModelEMA
    m = build_mirror("n", nc=15, seed=0).to(DEV)
    ref = copy.deepcopy(m)
    opt = _torch_adam(ref, betas)
    ema = ModelEMA(m)
    ema_ref = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    grads = {p: torch.zeros_like(p) for p in m.parameters()}
    fused = _fused(m, grads, ema.ema)
    gen = torch.Generator(device=DEV).manual_seed(0)
    for step in range(5):
        for (p, g), pr in zip(grads.items(), ref.parameters()):
            g.copy_(_grad(p.shape, gen))
            pr.grad = g.clone()
        with torch.no_grad():  # BatchNorm running statistics move during training: EMA follows them too
            for b, br in zip(m.buffers(), ref.buffers()):
                if b.dtype.is_floating_point:
                    b.add_(0.01)
                    br.add_(0.01)
        lr = _lrs(step)
        for grp, v in zip(opt.param_groups, lr):
            grp["lr"] = v
        opt.step()
        ema.updates += 1
        d = ema.decay(ema.updates)
        fused.step(lr, betas, 1e-8, d)
        with torch.no_grad():   # utils/torch_utils.py:304-314, per tensor: v *= d; v += (1 - d) * msd[k]
            msd = ref.state_dict()
            for k, v in ema_ref.items():
                if v.dtype.is_floating_point:
                    v *= d
                    v += (1 - d) * msd[k]
    torch.cuda.synchronize()
    for (n, a), b in zip(m.named_parameters(), ref.parameters()):
        assert torch.equal(a, b), n
        s, sr = fused.state[a], opt.state[b]
        assert torch.equal(s["exp_avg"], sr["exp_avg"]), n
        assert torch.equal(s["exp_avg_sq"], sr["exp_avg_sq"]), n
        assert float(s["step"]) == float(sr["step"]) == 5.0
    for k, a in ema.ema.state_dict().items():
        if a.dtype.is_floating_point:
            assert torch.equal(a, ema_ref[k]), k


def _run_train_steps(fused: str, n: int, x, tg, **kw):
    from yolov5_obb_b200.train_step import TrainStep
    os.environ["Y5OBB_FUSED_SGD"] = fused
    try:
        m = build_mirror("n", nc=15, seed=0).to(DEV).train()
        ts = TrainStep(m, imgsz=128, adam=True, **kw)
        for _ in range(n):
            ts.step(x, tg)
        torch.cuda.synchronize()
    finally:
        os.environ.pop("Y5OBB_FUSED_SGD", None)
    return m, ts


def _batch():
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    tg = torch.from_numpy(synth_targets(2, 12, 128, nc=15, seed=2)).to(DEV)
    return x, tg


def _rel(A, B):
    num = sum(((a - b).double() ** 2).sum().item() for a, b in zip(A, B)) ** 0.5
    den = sum((b.double() ** 2).sum().item() for b in B) ** 0.5
    return num / den


def test_train_step_adam_fused_equals_torch_path():
    """TrainStep(adam=True) with the fused kernel and with torch.optim.Adam + foreach EMA (Y5OBB_FUSED_SGD=0) from the same
    start: after 3 steps parameters, moments and EMA agree to rounding (the backward's split-K atomics make the two runs'
    gradients differ in the last bits)."""
    x, tg = _batch()
    res = []
    for fused in ("1", "0"):
        m, ts = _run_train_steps(fused, 3, x, tg, batch_size=64)
        assert ts._use_fused == (fused == "1")
        assert isinstance(ts.optimizer, torch.optim.Adam)
        st = [ts.optimizer.state[p] for p in m.parameters()]
        assert all(float(s["step"]) == 3.0 for s in st)
        res.append(([p.detach().clone() for p in m.parameters()], [s["exp_avg"].clone() for s in st],
                    [s["exp_avg_sq"].clone() for s in st],
                    [v.clone() for v in ts.ema.ema.state_dict().values() if v.dtype.is_floating_point], ts.ema.updates))
    (pa, ma, va, ea, ua), (pb, mb, vb, eb, ub) = res
    assert ua == ub == 3
    for name, A, B, tol in (("param", pa, pb, 2e-3), ("exp_avg", ma, mb, 5e-2), ("exp_avg_sq", va, vb, 5e-2),
                            ("ema", ea, eb, 2e-3)):
        assert _rel(A, B) < tol, (name, _rel(A, B))


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)   # train.py:389-393 saves optimizer.state_dict() inside the checkpoint
    buf.seek(0)
    return torch.load(buf, weights_only=False)


def test_checkpoint_resume_bit_equal():
    """3 fused steps, optimizer.state_dict() through torch.save / torch.load; then a fresh torch.optim.Adam and a new
    FusedAdamEMA that adopts the loaded state each take step 4: both equal 4 uninterrupted fused steps bit for bit."""
    betas = (0.937, 0.999)
    base = build_mirror("n", nc=15, seed=0).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    gseq = [[_grad(p.shape, gen) for p in base.parameters()] for _ in range(4)]

    def make(model, state=None):
        grads = {p: torch.zeros_like(p) for p in model.parameters()}
        return _fused(model, grads, state=state), grads

    def run(fg, steps):
        f, grads = fg
        for k in steps:
            for g, src in zip(grads.values(), gseq[k]):
                g.copy_(src)
            f.step(_lrs(k), betas, 1e-8)
        return f

    full = copy.deepcopy(base)
    ff = run(make(full), range(4))

    part = copy.deepcopy(base)
    fp = run(make(part), range(3))
    opt = _torch_adam(part, betas)
    for p, s in fp.state.items():   # what TrainStep registers
        opt.state[p] = s
    torch.cuda.synchronize()
    sd = _roundtrip(opt.state_dict())
    assert sorted(sd["state"][0]) == ["exp_avg", "exp_avg_sq", "step"]

    # (a) a fresh torch.optim.Adam takes step 4
    ma = copy.deepcopy(part)
    oa = _torch_adam(ma, betas)
    oa.load_state_dict(sd)
    for grp, v in zip(oa.param_groups, _lrs(3)):
        grp["lr"] = v
    for p, g in zip(ma.parameters(), gseq[3]):
        p.grad = g.clone()
    oa.step()
    # (b) a new FusedAdamEMA adopts the loaded state (of another fresh optimizer) and takes step 4
    mb = copy.deepcopy(part)
    ob = _torch_adam(mb, betas)
    ob.load_state_dict(_roundtrip(opt.state_dict()))
    fb, gb = make(mb, state=ob.state)
    assert fb.t == 3.0 and all(fb.state[p]["exp_avg"] is ob.state[p]["exp_avg"] for p in mb.parameters())
    run((fb, gb), [3])
    torch.cuda.synchronize()
    want = list(full.parameters())
    for model, st in ((ma, oa.state), (mb, fb.state)):
        for (n, a), b in zip(model.named_parameters(), want):
            assert torch.equal(a, b), n
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(st[a][k], ff.state[b][k]), (n, k)
            assert float(st[a]["step"]) == 4.0


def test_train_step_adam_resume_adopts_loaded_state():
    """TrainStep(adam=True): after optimizer.load_state_dict() of a 3-step checkpoint the next fused step runs on the
    loaded tensors (adopted in place) with step count 4, and agrees to rounding with the uninterrupted run's step 4."""
    from yolov5_obb_b200.train_step import TrainStep
    x, tg = _batch()
    m, ts = _run_train_steps("1", 3, x, tg, batch_size=64)
    sd = _roundtrip(ts.optimizer.state_dict())
    m2 = build_mirror("n", nc=15, seed=0).to(DEV).train()
    m2.load_state_dict(m.state_dict())
    ts2 = TrainStep(m2, batch_size=64, imgsz=128, adam=True)
    ts2.ema.ema.load_state_dict(ts.ema.ema.state_dict())
    ts2.ema.updates = ts.ema.updates
    ts2.optimizer.load_state_dict(sd)
    loaded = [ts2.optimizer.state[p]["exp_avg"] for p in m2.parameters()]
    ts.step(x, tg)
    ts2.step(x, tg)
    torch.cuda.synchronize()
    st2 = [ts2.optimizer.state[p] for p in m2.parameters()]
    assert all(s["exp_avg"] is t for s, t in zip(st2, loaded))
    assert all(float(s["step"]) == 4.0 for s in st2)
    st = [ts.optimizer.state[p] for p in m.parameters()]
    assert _rel(list(m2.parameters()), list(m.parameters())) < 2e-3
    assert _rel([s["exp_avg"] for s in st2], [s["exp_avg"] for s in st]) < 5e-2


def test_accumulation_runs_torch_adam_every_fourth_step():
    """batch_size=16: accumulate = 4, so torch.optim.Adam (not the fused kernel) runs and updates only on every fourth step."""
    x, tg = _batch()
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=0).to(DEV).train()
    ts = TrainStep(m, batch_size=16, imgsz=128, adam=True)
    assert ts.accumulate == 4 and not ts._use_fused and isinstance(ts.optimizer, torch.optim.Adam)
    p0 = [p.detach().clone() for p in m.parameters()]
    for i in range(4):
        ts.step(x, tg)
        torch.cuda.synchronize()
        same = all(torch.equal(a, b) for a, b in zip(m.parameters(), p0))
        assert same == (i < 3), i
    assert ts._fused is None and ts.ema.updates == 1
    assert all(float(ts.optimizer.state[p]["step"]) == 1.0 for p in m.parameters())


def test_run_refuses_bad_arguments():
    """y5obb_adam_ema_plan_run on a valid plan: betas outside [0, 1), a non-positive bc2_sqrt and a NULL step-size table are
    Y5OBB_EINVAL, and nothing is written."""
    from yolov5_obb_b200 import _lib
    m = build_mirror("n", nc=15, seed=0).to(DEV)
    grads = {p: torch.ones_like(p) for p in m.parameters()}
    f = _fused(m, grads)
    p0 = [p.detach().clone() for p in m.parameters()]
    L = _lib.lib()
    ss = (ctypes.c_float * 3)(-0.01, -0.01, -0.01)
    s = _lib.stream_ptr(DEV)
    for args in ((ss, 1.0, 0.999, 0.03, 1e-8), (ss, -0.1, 0.999, 0.03, 1e-8), (ss, 0.9, 1.0, 0.03, 1e-8),
                 (ss, 0.9, float("nan"), 0.03, 1e-8), (ss, 0.9, 0.999, 0.0, 1e-8), (ss, 0.9, 0.999, float("nan"), 1e-8),
                 (None, 0.9, 0.999, 0.03, 1e-8)):
        assert L.y5obb_adam_ema_plan_run(f._h, *args, 0.0, s) == 1, args
    assert L.y5obb_adam_ema_plan_run(None, ss, 0.9, 0.999, 0.03, 1e-8, 0.0, s) == 1
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(m.parameters(), p0))
    assert all(float(st["step"]) == 0.0 for st in f.state.values())
