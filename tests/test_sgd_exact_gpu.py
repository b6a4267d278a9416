"""Bit-exact checks of the SGD step (csrc/sgd_ema.cu k_sgd_ema, train_ops.FusedSGDEMA, TrainStep's fused path) against
torch.optim.SGD(nesterov=True)'s foreach step with the reference's parameter groups (train.py:148-162), and of every EMA the
project computes against the reference's per-tensor ModelEMA.update (utils/torch_utils.py:304-314), written out below.
Everything is compared with torch.equal: a step that drifts from torch in the last bit, or a wrong rule on a small term,
fails here.  Covered: warm-up learning rates and momenta that change every step, both EMA regimes (1 - d near 1 and
d near 1), table edges through the C ABI (tensor sizes around the 32- and 256-element boundaries, a tensor across the
grid-stride wrap), checkpoint resume at kernel level and through TrainStep, and the refusals of the C ABI and TrainStep."""
import copy
import ctypes
import gc
import io
import math
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
    the next module."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _lrs(step):
    """Per-group learning rates that change every step; step 0 is the warm-up's first: weights at 0, biases at 0.1."""
    return (0.0, 0.0, 0.1) if step == 0 else (0.002 * step, 0.003 * step, 0.1 - 0.015 * step)


def _mom(step, n=6):
    """The warm-up's momentum ramp from hyp['warmup_momentum'] 0.8 to hyp['momentum'] 0.937 over n steps."""
    return 0.8 + (0.937 - 0.8) * step / (n - 1)


def _grad(shape, gen):
    """Seeded gradients over six decades, with about 10 % exact zeros, 10 % values near 1e-30 and 5 % fp32 subnormals
    (near 1e-40)."""
    g = torch.randn(shape, generator=gen, device=DEV)
    g = g * 10.0 ** (torch.rand(shape, generator=gen, device=DEV) * 6 - 4)
    u = torch.rand(shape, generator=gen, device=DEV)
    g = torch.where(u < 0.1, torch.zeros_like(g), g)
    g = torch.where((u >= 0.1) & (u < 0.2), torch.randn(shape, generator=gen, device=DEV) * 1e-30, g)
    return torch.where((u >= 0.2) & (u < 0.25), torch.randn(shape, generator=gen, device=DEV) * 1e-40, g)


def _ema_rule(ema: dict, msd: dict, d: float):
    """utils/torch_utils.py:304-314, ModelEMA.update's loop body, on CUDA tensors: for every floating-point entry
    v *= d; v += (1 - d) * msd[k]."""
    with torch.no_grad():
        for k, v in ema.items():
            if v.dtype.is_floating_point:
                v *= d
                v += (1 - d) * msd[k].detach()


def _equal(a, b, what):
    assert a.shape == b.shape, what
    if not torch.equal(a, b):
        bad = int((a != b).sum())
        raise AssertionError(f"{what}: {bad} of {a.numel()} elements differ")


def _torch_sgd(params_by_group, momentum, lrs=(0.01, 0.01, 0.01), wds=(0.0, WD, 0.0)):
    g0, g1, g2 = params_by_group
    opt = torch.optim.SGD(g0, lr=lrs[0], momentum=momentum, nesterov=True, weight_decay=wds[0], foreach=True)
    opt.add_param_group({"params": g1, "lr": lrs[1], "weight_decay": wds[1]})
    opt.add_param_group({"params": g2, "lr": lrs[2], "weight_decay": wds[2]})
    return opt


def _set_groups(opt, lr, momentum=None):
    for grp, v in zip(opt.param_groups, lr):
        grp["lr"] = v
        if momentum is not None:
            grp["momentum"] = momentum


def _move_buffers(models, gen):
    """BatchNorm running statistics move during training: the EMA-only entries follow them."""
    with torch.no_grad():
        for bufs in zip(*[m.buffers() for m in models]):
            if bufs[0].dtype.is_floating_point:
                r = torch.rand(bufs[0].shape, generator=gen, device=DEV) * 0.1
                for b in bufs:
                    b.add_(r)


# ---- 1. FusedSGDEMA against torch.optim.SGD and the reference's EMA rule ---------------------------------------------------

@pytest.mark.parametrize("updates0", [0, 100_000])   # d about 5e-4 (1 - d near 1) and about 0.9999
def test_fused_sgd_bit_equal_to_torch_sgd_and_ema(updates0):
    from yolov5_obb_b200.train_ops import FusedSGDEMA
    from yolov5_obb_b200.train_step import ModelEMA, param_groups
    m = build_mirror("n", nc=15, seed=0).to(DEV)
    ref = copy.deepcopy(m)
    opt = _torch_sgd(param_groups(ref), _mom(0))
    ema = ModelEMA(m, updates=updates0)
    ema_ref = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    grads = {p: torch.zeros_like(p) for p in m.parameters()}
    fused = FusedSGDEMA(m, param_groups(m), grads, ema.ema, weight_decay=WD)
    gen = torch.Generator(device=DEV).manual_seed(0)
    for step in range(6):
        for (p, g), pr in zip(grads.items(), ref.parameters()):
            g.copy_(_grad(p.shape, gen))
            pr.grad = g.clone()
        _move_buffers((m, ref), gen)
        lr, mom = _lrs(step), _mom(step)
        _set_groups(opt, lr, mom)
        opt.step()
        ema.updates += 1
        d = ema.decay(ema.updates)
        fused.step(lr, mom, d)
        _ema_rule(ema_ref, ref.state_dict(), d)
        torch.cuda.synchronize()
        for (n, a), b in zip(m.named_parameters(), ref.parameters()):
            _equal(a, b, (step, n))
            _equal(fused.mom[a], opt.state[b]["momentum_buffer"], (step, n, "momentum_buffer"))
        for k, v in ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                _equal(v, ema_ref[k], (step, k, "ema"))
    assert 0.9998 < d if updates0 else d < 1e-2


# ---- 3. the torch path's ModelEMA ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("updates0,dtype", [(0, torch.float32), (100_000, torch.float32), (0, torch.float64)],
                         ids=["fp32-d5e-4", "fp32-d0.9999", "fp64-d5e-4"])
def test_model_ema_update_is_the_reference_rule(updates0, dtype):
    """train_step.ModelEMA.update (the EMA of every run with gradient accumulation, train.py's default batch of 16
    included) equals the reference's per-tensor rule bit for bit: fp32 through the EMA-only kernel table, other types
    through foreach ops."""
    from yolov5_obb_b200.train_step import ModelEMA
    m = build_mirror("n", nc=15, seed=0).to(DEV, dtype)
    ema = ModelEMA(m, updates=updates0)
    ema_ref = {k: v.clone() for k, v in ema.ema.state_dict().items()}
    gen = torch.Generator(device=DEV).manual_seed(3)
    for step in range(4):
        with torch.no_grad():
            for p in m.parameters():
                p.add_(_grad(p.shape, gen))
        _move_buffers((m,), gen)
        ema.update(m)
        _ema_rule(ema_ref, m.state_dict(), ema.decay(ema.updates))
        torch.cuda.synchronize()
        assert (ema._fused is not None) == (dtype == torch.float32)
        for k, v in ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                _equal(v, ema_ref[k], (step, k))


# ---- 4. table edges through the C ABI --------------------------------------------------------------------------------------

SIZES = (1, 2, 31, 32, 33, 255, 256, 257, 1023, 1025, 4097)
GAP = 5              # guard elements before, between and after the tensors of a flat buffer
SENTINEL = 12345.0


class _Table:
    """Tensors of the given sizes as views of guarded flat buffers (one per role), so a kernel that reads or writes one
    element past a tensor touches a guard of this buffer, which the checks compare, and never memory it does not own."""

    def __init__(self, sizes, roles, gen):
        self.sizes = sizes
        self.offs, o = [], GAP
        for n in sizes:
            self.offs.append(o)
            o += n + GAP
        self.flat = {r: torch.full((o,), SENTINEL, device=DEV) for r in roles}
        self.flat["p"].copy_(torch.randn(o, generator=gen, device=DEV))
        self.guard = torch.ones(o, dtype=torch.bool, device=DEV)
        for off, n in zip(self.offs, sizes):
            self.guard[off:off + n] = False
        self.initial = {r: t.clone() for r, t in self.flat.items()}

    def view(self, role, k):
        return self.flat[role][self.offs[k]:self.offs[k] + self.sizes[k]]

    def ptr(self, role, k):
        return self.view(role, k).data_ptr()

    def check_guards(self, what):
        for r, t in self.flat.items():
            _equal(t[self.guard], self.initial[r][self.guard], (what, r, "guard"))


def _edge_sizes():
    """SIZES, one tensor across the grid-stride wrap (grid_for: sm_count * 32 CTAs of 256 threads), SIZES reversed."""
    wrap = torch.cuda.get_device_properties(DEV).multi_processor_count * 32 * 256
    big = wrap - sum(SIZES) + 777            # starts before the wrap, ends 777 elements past it
    return list(SIZES) + [big] + list(SIZES[::-1]), len(SIZES)


def _edge_groups(n_entries):
    """Groups 0 / 1 / 2 / -1 in turn (the wrap tensor lands in group 1, with weight decay); every fifth trainable entry
    has no EMA."""
    groups = [(0, 1, 2, -1)[(k + 2) % 4] for k in range(n_entries)]
    has_ema = [g < 0 or k % 5 != 1 for k, g in enumerate(groups)]
    return groups, has_ema


def test_sgd_table_edges_through_the_c_abi():
    from yolov5_obb_b200 import _lib
    from yolov5_obb_b200.train_ops import SgdEntry
    sizes, wrap_k = _edge_sizes()
    groups, has_ema = _edge_groups(len(sizes))
    assert groups[wrap_k] == 1
    gen = torch.Generator(device=DEV).manual_seed(11)
    t = _Table(sizes, ("p", "g", "mom", "ema"), gen)
    t.flat["ema"].copy_(torch.where(t.guard, t.flat["ema"], torch.randn(t.flat["ema"].shape, generator=gen, device=DEV)))
    t.initial["ema"] = t.flat["ema"].clone()
    ent = []
    for k, (gk, e) in enumerate(zip(groups, has_ema)):
        tr = gk >= 0
        ent.append(SgdEntry(t.ptr("p", k), t.ptr("g", k) if tr else None, t.ptr("mom", k) if tr else None,
                            t.ptr("ema", k) if e else None, sizes[k], WD if gk == 1 else 0.0, gk))
    arr = (SgdEntry * len(ent))(*ent)
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.y5obb_sgd_ema_plan_create(arr, len(ent), ctypes.byref(h)) == 0
    try:
        ref_p = [t.view("p", k).clone() for k in range(len(sizes))]
        ref_e = {k: t.view("ema", k).clone() for k in range(len(sizes)) if has_ema[k]}
        opt = _torch_sgd([[ref_p[k] for k in range(len(sizes)) if groups[k] == j] for j in range(3)], _mom(0))
        for step in range(3):
            for k, gk in enumerate(groups):
                if gk >= 0:
                    t.view("g", k).copy_(_grad((sizes[k],), gen))
                    ref_p[k].grad = t.view("g", k).clone()
                else:   # an EMA-only entry: its tensor moves between steps, as BatchNorm statistics do
                    r = torch.randn(sizes[k], generator=gen, device=DEV)
                    t.view("p", k).add_(r)
                    ref_p[k].add_(r)
            lr, mom, d = _lrs(step), _mom(step), 0.9999 * (1 - math.exp(-(step + 1) / 2000))
            _set_groups(opt, lr, mom)
            opt.step()
            _ema_rule(ref_e, {k: ref_p[k] for k in ref_e}, d)
            lr3 = (ctypes.c_float * 3)(*lr)
            assert L.y5obb_sgd_ema_plan_run(h, lr3, mom, d, int(step == 0), _lib.stream_ptr(DEV)) == 0
            torch.cuda.synchronize()
            for k, gk in enumerate(groups):
                what = (step, k, sizes[k], gk)
                _equal(t.view("p", k), ref_p[k], what)
                if gk >= 0:
                    _equal(t.view("mom", k), opt.state[ref_p[k]]["momentum_buffer"], what + ("momentum_buffer",))
                if has_ema[k]:
                    _equal(t.view("ema", k), ref_e[k], what + ("ema",))
                else:
                    _equal(t.view("ema", k), t.initial["ema"][t.offs[k]:t.offs[k] + sizes[k]], what + ("no ema",))
            t.check_guards(step)
    finally:
        L.y5obb_sgd_ema_plan_destroy(h)


def test_adam_table_edges_through_the_c_abi():
    from yolov5_obb_b200 import _lib
    from yolov5_obb_b200.train_ops import AdamEntry, adam_step_scalars
    sizes, wrap_k = _edge_sizes()
    groups, has_ema = _edge_groups(len(sizes))
    gen = torch.Generator(device=DEV).manual_seed(12)
    t = _Table(sizes, ("p", "g", "m", "v", "ema"), gen)
    for r in ("m", "v", "ema"):
        t.flat[r].copy_(torch.where(t.guard, t.flat[r], torch.zeros_like(t.flat[r])))
    t.flat["ema"].copy_(torch.where(t.guard, t.flat["ema"], t.flat["p"]))
    t.initial = {r: x.clone() for r, x in t.flat.items()}
    ent = []
    for k, (gk, e) in enumerate(zip(groups, has_ema)):
        tr = gk >= 0
        ent.append(AdamEntry(t.ptr("p", k), t.ptr("g", k) if tr else None, t.ptr("m", k) if tr else None,
                             t.ptr("v", k) if tr else None, t.ptr("ema", k) if e else None, sizes[k],
                             WD if gk == 1 else 0.0, gk))
    arr = (AdamEntry * len(ent))(*ent)
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.y5obb_adam_ema_plan_create(arr, len(ent), ctypes.byref(h)) == 0
    betas, eps = (0.937, 0.999), 1e-8
    try:
        ref_p = [t.view("p", k).clone() for k in range(len(sizes))]
        ref_e = {k: t.view("ema", k).clone() for k in range(len(sizes)) if has_ema[k]}
        by_group = [[ref_p[k] for k in range(len(sizes)) if groups[k] == j] for j in range(3)]
        opt = torch.optim.Adam(by_group[0], lr=0.01, betas=betas, eps=eps, foreach=True)
        opt.add_param_group({"params": by_group[1], "weight_decay": WD})
        opt.add_param_group({"params": by_group[2]})
        for step in range(3):
            for k, gk in enumerate(groups):
                if gk >= 0:
                    t.view("g", k).copy_(_grad((sizes[k],), gen))
                    ref_p[k].grad = t.view("g", k).clone()
                else:
                    r = torch.randn(sizes[k], generator=gen, device=DEV)
                    t.view("p", k).add_(r)
                    ref_p[k].add_(r)
            lr, d = _lrs(step), 0.9999 * (1 - math.exp(-(100_000 + step) / 2000))
            _set_groups(opt, lr)
            opt.step()
            _ema_rule(ref_e, {k: ref_p[k] for k in ref_e}, d)
            scal = [adam_step_scalars(v, betas[0], betas[1], float(step + 1)) for v in lr]
            ss = (ctypes.c_float * 3)(*[s for s, _ in scal])
            assert L.y5obb_adam_ema_plan_run(h, ss, betas[0], betas[1], scal[0][1], eps, d, _lib.stream_ptr(DEV)) == 0
            torch.cuda.synchronize()
            for k, gk in enumerate(groups):
                what = (step, k, sizes[k], gk)
                _equal(t.view("p", k), ref_p[k], what)
                if gk >= 0:
                    st = opt.state[ref_p[k]]
                    _equal(t.view("m", k), st["exp_avg"], what + ("exp_avg",))
                    _equal(t.view("v", k), st["exp_avg_sq"], what + ("exp_avg_sq",))
                if has_ema[k]:
                    _equal(t.view("ema", k), ref_e[k], what + ("ema",))
                else:
                    _equal(t.view("ema", k), t.initial["ema"][t.offs[k]:t.offs[k] + sizes[k]], what + ("no ema",))
            t.check_guards(step)
    finally:
        L.y5obb_adam_ema_plan_destroy(h)


# ---- 5. checkpoint resume at kernel level ----------------------------------------------------------------------------------

def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)   # train.py:389-393 saves optimizer.state_dict() inside the checkpoint
    buf.seek(0)
    return torch.load(buf, weights_only=False)


def test_checkpoint_resume_bit_equal():
    """3 fused steps, optimizer.state_dict() through torch.save / torch.load; then a fresh torch.optim.SGD and a new
    FusedSGDEMA that adopts the loaded buffers each take step 4: both equal 4 uninterrupted fused steps bit for bit."""
    from yolov5_obb_b200.train_ops import FusedSGDEMA
    from yolov5_obb_b200.train_step import param_groups
    base = build_mirror("n", nc=15, seed=0).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(5)
    gseq = [[_grad(p.shape, gen) for p in base.parameters()] for _ in range(4)]

    def make(model, state=None):
        grads = {p: torch.zeros_like(p) for p in model.parameters()}
        return FusedSGDEMA(model, param_groups(model), grads, weight_decay=WD, state=state), grads

    def run(fg, steps):
        f, grads = fg
        for k in steps:
            for g, src in zip(grads.values(), gseq[k]):
                g.copy_(src)
            f.step(_lrs(k), _mom(k, 4))
        return f

    full = copy.deepcopy(base)
    ff = run(make(full), range(4))

    part = copy.deepcopy(base)
    fp = run(make(part), range(3))
    opt = _torch_sgd(param_groups(part), _mom(2, 4))
    for p, m in fp.mom.items():   # what TrainStep registers
        opt.state[p]["momentum_buffer"] = m
    torch.cuda.synchronize()
    sd = _roundtrip(opt.state_dict())
    assert sorted(sd["state"][0]) == ["momentum_buffer"]

    # (a) a fresh torch.optim.SGD takes step 4
    ma = copy.deepcopy(part)
    oa = _torch_sgd(param_groups(ma), 0.5)
    oa.load_state_dict(sd)
    _set_groups(oa, _lrs(3), _mom(3, 4))
    for p, g in zip(ma.parameters(), gseq[3]):
        p.grad = g.clone()
    oa.step()
    # (b) a new FusedSGDEMA adopts the loaded buffers (of another fresh optimizer) in place and takes step 4
    mb = copy.deepcopy(part)
    ob = _torch_sgd(param_groups(mb), 0.5)
    ob.load_state_dict(_roundtrip(opt.state_dict()))
    fb, gb = make(mb, state=ob.state)
    assert fb.steps == 1 and all(fb.mom[p] is ob.state[p]["momentum_buffer"] for p in mb.parameters())
    run((fb, gb), [3])
    torch.cuda.synchronize()
    want = list(full.parameters())
    for model, bufs in ((ma, {p: oa.state[p]["momentum_buffer"] for p in ma.parameters()}), (mb, fb.mom)):
        for (n, a), b in zip(model.named_parameters(), want):
            _equal(a, b, n)
            _equal(bufs[a], ff.mom[b], (n, "momentum_buffer"))


# ---- 6, 7. TrainStep: resume, and the fused step against the torch path on the same gradient ------------------------------

def _batch():
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    tg = torch.from_numpy(synth_targets(2, 12, 128, nc=15, seed=2)).to(DEV)
    return x, tg


def _snapshot(ts):
    m, opt = ts.model, ts.optimizer
    return dict(params=[p.detach().clone() for p in m.parameters()],
                bufs=[opt.state[p]["momentum_buffer"].clone() if "momentum_buffer" in opt.state.get(p, {}) else None
                      for p in m.parameters()],
                ema={k: v.clone() for k, v in ts.ema.ema.state_dict().items()}, updates=ts.ema.updates)


def _check_step_exact(ts, pre):
    """After a fused TrainStep step: torch.optim.SGD applied to clones of the pre-step parameters and buffers with the
    gradient the step consumed (the backward plan's flat buffer), and the EMA rule on the pre-step EMA, equal the step's
    results bit for bit."""
    m, opt = ts.model, ts.optimizer
    params = list(m.parameters())
    pgrad = m._last_train_engine._bwd.pgrad
    q = [t.clone() for t in pre["params"]]
    idx = {id(p): i for i, p in enumerate(params)}
    g = opt.param_groups
    ref = _torch_sgd([[q[idx[id(p)]] for p in grp["params"]] for grp in g], g[0]["momentum"],
                     lrs=[grp["lr"] for grp in g], wds=[grp["weight_decay"] for grp in g])
    for p, qq, b in zip(params, q, pre["bufs"]):
        qq.grad = pgrad[p].clone()
        if b is not None:
            ref.state[qq]["momentum_buffer"] = b.clone()
    ref.step()
    ema = pre["ema"]
    _ema_rule(ema, m.state_dict(), ts.ema.decay(ts.ema.updates))
    assert ts.ema.updates == pre["updates"] + 1
    for (n, p), qq in zip(m.named_parameters(), q):
        _equal(p, qq, n)
        _equal(opt.state[p]["momentum_buffer"], ref.state[qq]["momentum_buffer"], (n, "momentum_buffer"))
    for k, v in ts.ema.ema.state_dict().items():
        if v.dtype.is_floating_point:
            _equal(v, ema[k], (k, "ema"))


def _train_step(m, **kw):
    from yolov5_obb_b200.train_step import TrainStep
    ts = TrainStep(m, batch_size=64, imgsz=128, **kw)
    assert ts.accumulate == 1 and ts._use_fused
    return ts


def test_train_step_resume_runs_on_the_loaded_momentum():
    """TrainStep: 3 steps, optimizer.state_dict() through torch.save / torch.load into a fresh TrainStep (EMA and updates
    copied as train.py:188-189 does).  The next step runs on the loaded momentum_buffer tensors, not as a first step, and
    equals torch.optim.SGD on its own gradient bit for bit; so does the step after a load_state_dict() mid-run."""
    x, tg = _batch()
    m = build_mirror("n", nc=15, seed=0).to(DEV).train()
    ts = _train_step(m)
    for _ in range(3):
        ts.step(x, tg)
    torch.cuda.synchronize()
    sd = _roundtrip(ts.optimizer.state_dict())
    m2 = build_mirror("n", nc=15, seed=0).to(DEV).train()
    m2.load_state_dict(m.state_dict())
    ts2 = _train_step(m2)
    ts2.ema.ema.load_state_dict(ts.ema.ema.state_dict())
    ts2.ema.updates = ts.ema.updates
    for sd_k in (sd, None):
        if sd_k is None:   # mid-run: a checkpoint of other buffers (the first run's, one step behind) is loaded
            ts.step(x, tg)
            torch.cuda.synchronize()
            sd_k = _roundtrip(ts.optimizer.state_dict())
        ts2.optimizer.load_state_dict(sd_k)
        params = list(m2.parameters())
        loaded = [ts2.optimizer.state[p]["momentum_buffer"] for p in params]
        assert all(b is not None and not b.eq(0).all() for b in loaded)
        pre = _snapshot(ts2)
        ts2.step(x, tg)
        torch.cuda.synchronize()
        assert all(ts2.optimizer.state[p]["momentum_buffer"] is b for p, b in zip(params, loaded))
        _check_step_exact(ts2, pre)


def test_train_step_fused_equals_torch_path_on_the_same_gradient():
    """After each fused TrainStep step (warm-up: lr and momentum change every step), the torch path's own update -
    TrainStep's torch.optim.SGD step and ModelEMA.update - applied to a snapshot of the pre-step state with .grad set to the
    gradients the fused step consumed gives the same parameters, momentum buffers and EMA bit for bit."""
    x, tg = _batch()
    m = build_mirror("n", nc=15, seed=0).to(DEV).train()
    ts = _train_step(m, warmup_iters=4)
    mt = build_mirror("n", nc=15, seed=0).to(DEV).train()
    from yolov5_obb_b200.train_step import TrainStep
    os.environ["Y5OBB_FUSED_SGD"] = "0"
    try:
        tt = TrainStep(mt, batch_size=64, imgsz=128, warmup_iters=4)
    finally:
        os.environ.pop("Y5OBB_FUSED_SGD", None)
    assert not tt._use_fused
    for step in range(3):
        pre = _snapshot(ts)
        ts.step(x, tg)
        torch.cuda.synchronize()
        pgrad = m._last_train_engine._bwd.pgrad
        mt.load_state_dict(m.state_dict())   # this step's BatchNorm statistics ...
        tt.optimizer.state.clear()
        with torch.no_grad():
            for p, pt, v, b in zip(m.parameters(), mt.parameters(), pre["params"], pre["bufs"]):
                pt.copy_(v)                   # ... and the pre-step parameters
                pt.grad = pgrad[p].clone()
                if b is not None:
                    tt.optimizer.state[pt]["momentum_buffer"] = b.clone()
        for gt, g in zip(tt.optimizer.param_groups, ts.optimizer.param_groups):
            gt["lr"], gt["momentum"] = g["lr"], g["momentum"]
            assert gt["weight_decay"] == g["weight_decay"]
        tt.ema.ema.load_state_dict(pre["ema"])
        tt.ema.updates = pre["updates"]
        tt.optimizer.step()
        tt.ema.update(mt)
        torch.cuda.synchronize()
        assert (pre["bufs"][0] is None) == (step == 0)
        for (n, a), b in zip(m.named_parameters(), mt.parameters()):
            _equal(a, b, (step, n))
            _equal(ts.optimizer.state[a]["momentum_buffer"], tt.optimizer.state[b]["momentum_buffer"], (step, n, "buf"))
        eb = tt.ema.ema.state_dict()
        for k, v in ts.ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                _equal(v, eb[k], (step, k, "ema"))
    assert len({g["momentum"] for g in ts.optimizer.param_groups}) == 1 and ts.optimizer.param_groups[0]["momentum"] < 0.937


# ---- 8. refusals -----------------------------------------------------------------------------------------------------------

def test_run_and_create_refuse_bad_arguments():
    """y5obb_sgd_ema_plan_run with a NULL lr table, a NaN or negative momentum or an EMA decay outside [0, 1], and
    y5obb_adam_ema_plan_run with such a decay, are Y5OBB_EINVAL and write nothing; y5obb_sgd_ema_plan_create refuses an
    EMA-only entry without an EMA."""
    from yolov5_obb_b200 import _lib
    from yolov5_obb_b200.train_ops import FusedAdamEMA, FusedSGDEMA, SgdEntry
    from yolov5_obb_b200.train_step import ModelEMA, param_groups
    m = build_mirror("n", nc=15, seed=0).to(DEV)
    ema = ModelEMA(m)
    with torch.no_grad():
        for v in ema.ema.state_dict().values():
            if v.dtype.is_floating_point:
                v.add_(1.0)
    grads = {p: torch.ones_like(p) for p in m.parameters()}
    f = FusedSGDEMA(m, param_groups(m), grads, ema.ema, weight_decay=WD)
    fa = FusedAdamEMA(m, param_groups(m), grads, ema.ema, weight_decay=WD)
    p0 = [p.detach().clone() for p in m.parameters()]
    e0 = [v.clone() for v in ema.ema.state_dict().values()]
    L = _lib.lib()
    s = _lib.stream_ptr(DEV)
    lr3 = (ctypes.c_float * 3)(0.01, 0.01, 0.01)
    nan = float("nan")
    for args in ((None, 0.9, 0.5, 0), (lr3, nan, 0.5, 0), (lr3, -0.1, 0.5, 0), (lr3, 0.9, -1e-9, 0), (lr3, 0.9, 1.5, 0),
                 (lr3, 0.9, nan, 1), (lr3, 0.9, float("inf"), 1)):
        assert L.y5obb_sgd_ema_plan_run(f._h, *args, s) == 1, args
    assert L.y5obb_sgd_ema_plan_run(None, lr3, 0.9, 0.5, 0, s) == 1
    ss = (ctypes.c_float * 3)(-0.01, -0.01, -0.01)
    for d in (-0.5, 1.0 + 1e-12, nan):
        assert L.y5obb_adam_ema_plan_run(fa._h, ss, 0.9, 0.999, 0.03, 1e-8, d, s) == 1, d
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(m.parameters(), p0))
    assert all(torch.equal(a, b) for a, b in zip(ema.ema.state_dict().values(), e0))
    assert all(not b.any() for b in f.mom.values())
    assert all(not st["exp_avg"].any() for st in fa.state.values())
    p = next(m.parameters())
    h = ctypes.c_void_p()
    for ent in (SgdEntry(p.data_ptr(), None, None, None, p.numel(), 0.0, -1),
                SgdEntry(p.data_ptr(), grads[p].data_ptr(), f.mom[p].data_ptr(), None, p.numel(), 0.0, 3)):
        assert L.y5obb_sgd_ema_plan_create((SgdEntry * 1)(ent), 1, ctypes.byref(h)) == 1
    # the edges of the accepted ranges run
    for d in (0.0, 1.0):
        assert L.y5obb_sgd_ema_plan_run(f._h, lr3, 0.0, d, 1, s) == 0


def test_train_step_refuses_group_momenta_that_differ():
    """The fused TrainStep step uses one momentum for every group: groups whose momenta differ are refused, naming the
    switch to torch.optim.SGD, instead of stepping every group with group 0's."""
    x, tg = _batch()
    m = build_mirror("n", nc=15, seed=0).to(DEV).train()
    ts = _train_step(m)
    ts.optimizer.param_groups[2]["momentum"] = 0.5
    p0 = [p.detach().clone() for p in m.parameters()]
    with pytest.raises(ValueError, match="Y5OBB_FUSED_SGD=0"):
        ts.step(x, tg)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(m.parameters(), p0))
