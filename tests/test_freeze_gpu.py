"""train.py --freeze on the device: the backward plan built for a set of frozen parameters (its launches against the full
plan's, its gradients against the full plan's), the windowed data-gradient weight pack, and TrainStep(freeze=...) with the
fused SGD / Adam + EMA step against the torch optimizers."""
import copy
import ctypes
import gc
import inspect
import os

import pytest
import torch

from tests.lossgen import synth_targets
from tests.modelgen import build_mirror
from yolov5_obb_b200.conv import Slice
from yolov5_obb_b200.layout import grad_liveness, shapes, sources
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainEngine, _PoolLayer
from yolov5_obb_b200.train_step import TrainStep, freeze_layers

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, H, W = 2, 256, 256


@pytest.fixture(autouse=True)
def _release():
    """Plans hold device buffers in reference cycles (their launch closures): free them when each test ends."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _engine(freeze):
    m = build_mirror("s", nc=15, seed=0).train().to(DEV)
    freeze_layers(m, freeze)
    eng = TrainEngine(m, B, H, W, DEV)
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        outs = eng.forward(x)
    g = torch.Generator().manual_seed(2)
    G = [(torch.randn(o.shape, generator=g) * 0.05).to(DEV) for o in outs]
    return m, eng, x, G


def _flags(m):
    return tuple(p.requires_grad for p in m.parameters())


def _defaults(fn):
    return {k: p.default for k, p in inspect.signature(fn).parameters.items() if p.default is not inspect.Parameter.empty}


def _norm(v):
    """A launch argument without its addresses: buffers by shape and channel window, layers by identity."""
    if isinstance(v, Slice):
        return ("slice", tuple(v.buf.shape), v.c_off, v.C)
    if isinstance(v, torch.Tensor):
        return ("tensor", tuple(v.shape), v.dtype)
    if isinstance(v, (int, float, bool, str)) or v is None:
        return v
    return ("obj", id(v))


def _desc(d):
    """A ctypes descriptor's fields other than addresses."""
    return tuple((n, getattr(d, n) if not hasattr(getattr(d, n), "__len__") else tuple(getattr(d, n)))
                 for n, t in d._fields_ if t is not ctypes.c_void_p)


def _ops(plan):
    ops = {}
    for part in plan.det_parts + plan.conv_parts:
        for op in part.get("dgrad_ops", ()):
            ops[op._h.value] = (op, part)
    return ops


def _sig(plan, tag, fn):
    a = _defaults(fn)
    if tag == "dgrad":
        op, _ = _ops(plan)[a["h"].value]
        info = op.info()
        return tag, _desc(op.desc), tuple(sorted(info.items()))
    if tag == "wgrad":
        return tag, _desc(a["wg"].desc)
    # (pool_bwd takes its gradient buffer as a bare address, "gbase")
    return tag, tuple(sorted((k, _norm(v)) for k, v in a.items() if k != "gbase"))


def _owner(m, eng, plan, tag, fn):
    """-> (kind, layer index, module, level) of a full-plan step."""
    a = _defaults(fn)
    top = {}
    for mm in m.model:
        for sub in mm.modules():
            top.setdefault(id(sub), mm.i)
    det = m.model[-1]
    if tag in ("detect_pack", "detect_bias"):
        lv = a["l"] if "l" in a else next(p["l"] for p in plan.det_parts if p["dzd"] is a["dzd"])
        return tag, det.i, det, lv
    if tag == "pool_bwd":
        pool = next(l for l in eng.layers if isinstance(l, _PoolLayer) and l.cat4.data_ptr() == a["base"])
        sppf = next(mm for mm in m.model if type(mm).__name__ == "SPPF")
        return tag, sppf.i, pool, None
    if tag == "wgrad":
        part = next(p for p in plan.det_parts + plan.conv_parts if p.get("wgrad") is a["wg"])
    elif tag == "dgrad":
        part = _ops(plan)[a["h"].value][1]
    elif tag == "zero":
        part = next(p for p in plan.conv_parts if p.get("stem_dw") is a["dw"])
    elif tag == "bn_bwd":
        part = next(p for p in plan.conv_parts if p["lay"] is a["lay"])
    else:   # upsample_bwd
        gy = a["gy"]
        part = next(p for p in plan.conv_parts
                    if plan.gbuf.get(p["lay"].y.buf.data_ptr()) is gy.buf and p["lay"].y.c_off == gy.c_off)
    if "mi" in part:
        return tag, det.i, part["mi"], part["l"]
    mod = part["lay"].mod
    return tag, top[id(mod)], mod, None


def _expected_keep(m, owner, need, windows, ch):
    """The liveness rule applied to one launch of the full plan, from the model-level liveness: True (kept), False
    (removed) or "window" (a dgrad kept for the live channel window of a Concat only)."""
    tag, i, mod, lv = owner
    mods = list(m.model)
    det = mods[-1]
    if type(mod).__name__ == "Conv2d" or tag in ("detect_pack", "detect_bias"):   # a Detect level
        det_tr = any(p.requires_grad for p in det.parameters())
        src_live = det.f[lv] in need
        return {"detect_pack": det_tr or src_live, "detect_bias": det_tr, "wgrad": det_tr, "dgrad": src_live}[tag]
    if i not in need:
        return False
    if tag in ("wgrad", "zero"):
        return mod.conv.weight.requires_grad
    if tag != "dgrad":
        return True
    top = mods[i]
    kind = type(top).__name__
    # the convs that read the layer's input: a Conv layer itself, a C3's cv1 / cv2, an SPPF's cv1
    if not (mod is top or (kind == "C3" and mod in (top.cv1, top.cv2)) or (kind == "SPPF" and mod is top.cv1)):
        return True   # (inside a needed layer every producer is live)
    src = sources(top)[0]
    if src not in need:
        return False
    return True if src not in windows or windows[src] == [(0, ch[src])] else "window"


@pytest.mark.parametrize("freeze", [[10], [0, 1, 2], [24], [5, 7], [0]])
def test_pruned_plan_is_a_subsequence_of_the_full_plan(freeze):
    m, eng, _, _ = _engine(freeze)
    full = BackwardPlan(eng)
    pruned = BackwardPlan(eng, _flags(m))
    mods = list(m.model)
    ch, _ = shapes(mods, H, W)
    need, windows = grad_liveness(mods, ch, lambda mm: any(p.requires_grad for p in mm.parameters()))
    if freeze == [0]:
        assert [_sig(full, t, f) for t, f in full.steps] == [_sig(pruned, t, f) for t, f in pruned.steps]
        return
    want = []
    for tag, fn in full.steps:
        k = _expected_keep(m, _owner(m, eng, full, tag, fn), need, windows, ch)
        if k:
            want.append((k, tag, fn))
    assert len(want) == len(pruned.steps), (len(want), len(pruned.steps), len(full.steps))
    n_win = 0
    for (k, tag, fn), (ptag, pfn) in zip(want, pruned.steps):
        assert tag == ptag
        if k == "window":     # the same dgrad conv, its output the live window of the gradient buffer
            op, part = _ops(pruned)[_defaults(pfn)["h"].value]
            x = part["lay"].x
            (c0, n, _), = part["dgrad_win"]
            src = sources(mods[_owner(m, eng, pruned, ptag, pfn)[1]])[0]
            assert x.c_off == 0 and x.C == ch[src] and windows[src] == [(c0, c0 + n)] and n < x.C
            assert op.desc.Cout == n and op.desc.out == pruned.gbuf[x.buf.data_ptr()].data_ptr() + 2 * c0
            n_win += 1
            continue
        assert _sig(full, tag, fn) == _sig(pruned, ptag, pfn), tag
    assert n_win == (4 if freeze == [10] else 0)   # 13.cv1, 13.cv2, 17.cv1, 17.cv2
    if freeze == [10]:
        assert all(_owner(m, eng, pruned, t, f)[1] >= 10 for t, f in pruned.steps)


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("freeze", [[10], [0, 1, 2], [24], [5, 7]])
def test_pruned_plan_gradients_equal_the_full_plans(freeze):
    m, eng, x, G = _engine(freeze)
    full = BackwardPlan(eng)

    def run(plan):
        plan.run(G)
        torch.cuda.synchronize()
        return {k: t.clone() for k, t in plan.gbuf.items()}, {p: plan.pgrad[p].clone() for p in plan.params}

    f1, f2 = run(full), run(full)
    pruned = BackwardPlan(eng, _flags(m))
    pr = run(pruned)
    # the full plan's run-to-run spread (split-K and reduction atomics reorder fp32 sums)
    spread_buf = max(_rel(a, f1[0][k]) for k, a in f2[0].items())
    spread_par = max(_rel(a, f1[1][p]) for p, a in f2[1].items())
    acts = {t.data_ptr(): t for t in eng.keep}
    checked = 0
    for k, g in pr[0].items():
        for lo, hi in pruned.live_windows(Slice.full(acts[k])):
            a, b = g[..., lo:hi].float(), f1[0][k][..., lo:hi].float()
            if spread_buf == 0:
                assert torch.equal(a, b), (k, lo, hi)
            else:
                assert _rel(a, b) <= 2 * spread_buf, (k, lo, hi, _rel(a, b), spread_buf)
            checked += 1
    assert (checked > 0) == (freeze != [24])   # [24]: only Detect trains, no data gradient is needed
    for p, t in zip(m.parameters(), pruned.trainable):
        if not t:
            continue
        if spread_par == 0:
            assert torch.equal(pr[1][p], f1[1][p])
        else:
            assert _rel(pr[1][p], f1[1][p]) <= 2 * spread_par + 1e-7, (_rel(pr[1][p], f1[1][p]), spread_par)
    # through autograd: a frozen parameter's .grad stays None
    outs = m(x)
    sum((o * g).sum() for o, g in zip(outs, G)).backward()
    for p in m.parameters():
        assert (p.grad is None) == (not p.requires_grad)


def test_windowed_dgrad_pack():
    """PACK_DGRAD over the channel window [c0, c0 + n) equals PACK_DGRAD of the window's contiguous copy, byte for byte."""
    from yolov5_obb_b200.conv import pack_weights
    from yolov5_obb_b200.train_ops import PackPlan, PACK_DGRAD, PACK_DGRAD_S2
    g = torch.Generator(device=DEV).manual_seed(3)
    for cout, cin, k, c0, n in ((128, 256, 1, 0, 128), (128, 256, 1, 128, 128), (64, 200, 3, 40, 72), (96, 48, 1, 0, 48)):
        w = torch.randn((cout, cin, k, k), device=DEV, generator=g)
        got = pack_weights(torch.zeros((n, cout, k, k), device=DEV), None)[0].fill_(7)
        ref = pack_weights(torch.zeros((n, cout, k, k), device=DEV), None)[0].fill_(-7)
        PackPlan([(PACK_DGRAD, w, got, c0, n)], DEV).run()
        PackPlan([(PACK_DGRAD, w[:, c0:c0 + n].contiguous(), ref, 0, 0)], DEV).run()
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16)), (cout, cin, k, c0, n)
    w = torch.randn((64, 32, 3, 3), device=DEV, generator=g)
    dst = pack_weights(torch.zeros((16, 64, 3, 3), device=DEV), None)[0]
    for kind, gr, gp in ((PACK_DGRAD, 24, 16), (PACK_DGRAD, 8, 0), (PACK_DGRAD, -1, 8), (PACK_DGRAD_S2, 0, 16)):
        with pytest.raises(RuntimeError):
            PackPlan([(kind, w, dst if kind == PACK_DGRAD else pack_weights(torch.zeros((32, 64, 1, 1), device=DEV), None)[0],
                       gr, gp)], DEV)


def _batch():
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    tg = torch.from_numpy(synth_targets(2, 12, 128, nc=15, seed=2)).to(DEV)
    return x, tg


def _run(fused, adam, freeze, steps, unfreeze_after=None, multi_scale=False):
    os.environ["Y5OBB_FUSED_SGD"] = fused
    try:
        x, tg = _batch()
        m = build_mirror("n", nc=15, seed=0).to(DEV).train()
        ts = TrainStep(m, batch_size=64, imgsz=128, adam=adam, freeze=freeze, multi_scale=multi_scale, seed=0)
        start = [p.detach().clone() for p in m.parameters()]
        for i in range(steps):
            if unfreeze_after is not None and i == unfreeze_after:
                for p in m.parameters():
                    p.requires_grad_(True)
            ts.step(x, tg)
        torch.cuda.synchronize()
        return m, ts, start
    finally:
        os.environ.pop("Y5OBB_FUSED_SGD", None)


def _total_rel(A, B):
    num = sum(((a - b).double() ** 2).sum().item() for a, b in zip(A, B)) ** 0.5
    den = sum((b.double() ** 2).sum().item() for b in B) ** 0.5
    return num / den


@pytest.mark.parametrize("adam", [False, True])
def test_train_step_freeze_fused_equals_torch_path(adam):
    runs = [_run(f, adam, [10], 3) for f in ("1", "0")]
    (ma, tsa, sa), (mb, tsb, sb) = runs
    assert tsa._use_fused and not tsb._use_fused
    frozen = [i for i, p in enumerate(ma.parameters()) if not p.requires_grad]
    assert frozen and [i for i, p in enumerate(mb.parameters()) if not p.requires_grad] == frozen
    pa, pb = list(ma.parameters()), list(mb.parameters())
    for i in frozen:   # not moved by gradient, weight decay or momentum
        assert torch.equal(pa[i], sa[i]) and torch.equal(pb[i], sb[i]), i
    # the frozen parameters' EMA entries equal ModelEMA's (the torch path's): both round as the reference's per-tensor ops
    names = {n for n, p in ma.named_parameters() if not p.requires_grad}
    ea, eb = tsa.ema.ema.state_dict(), tsb.ema.ema.state_dict()
    for n in names:
        assert torch.equal(ea[n], eb[n]), n
    assert tsa.ema.updates == tsb.ema.updates == 3
    train = [i for i in range(len(pa)) if i not in frozen]
    assert _total_rel([pa[i] for i in train], [pb[i] for i in train]) < 2e-3
    assert _total_rel([v for v in ea.values() if v.dtype.is_floating_point],
                      [v for v in eb.values() if v.dtype.is_floating_point]) < 2e-3
    for ts, m in ((tsa, ma), (tsb, mb)):
        for i in frozen:
            assert list(m.parameters())[i] not in ts.optimizer.state
    # the fused path's state loads into the plain torch optimizer
    sd = copy.deepcopy(tsa.optimizer.state_dict())
    g = [g_["params"] for g_ in tsb.optimizer.param_groups]
    opt = (torch.optim.Adam if adam else torch.optim.SGD)(g[0], lr=0.01)
    for p in g[1:]:
        opt.add_param_group({"params": p})
    opt.load_state_dict(sd)
    assert len(opt.state) == len(train)


@pytest.mark.parametrize("adam", [False, True])
def test_unfreeze_mid_run(adam):
    """[10] for 2 steps, then every parameter trainable for 2 more: the fused path against torch's optimizer doing the same."""
    (ma, tsa, _), (mb, tsb, _) = [_run(f, adam, [10], 4, unfreeze_after=2) for f in ("1", "0")]
    assert tsa._use_fused == (not adam)     # Adam leaves the fused step after an unfreeze
    eng = ma._last_train_engine
    assert len(eng._bwds) == 2 and all(eng._bwd.trainable)
    # Adam's first step moves every element of a newly trainable parameter by about lr * sign(grad), however small the
    # gradient: the last-bit gradient differences of the two runs flip the sign of near-zero elements, hence the wider bound
    tol = 3e-2 if adam else 2e-3
    assert _total_rel(list(ma.parameters()), list(mb.parameters())) < tol
    ea = [v for v in tsa.ema.ema.state_dict().values() if v.dtype.is_floating_point]
    eb = [v for v in tsb.ema.ema.state_dict().values() if v.dtype.is_floating_point]
    assert _total_rel(ea, eb) < tol
    if adam:   # (the moments of the newly trainable elements inherit the same sign flips: their step counts are compared)
        steps = {float(tsb.optimizer.state[p]["step"]) for p in mb.parameters()}
        assert steps == {2.0, 4.0} == {float(tsa.optimizer.state[p]["step"]) for p in ma.parameters()}
    else:
        sa = [tsa.optimizer.state[p]["momentum_buffer"] for p in ma.parameters()]
        sb = [tsb.optimizer.state[p]["momentum_buffer"] for p in mb.parameters()]
        assert _total_rel(sa, sb) < 5e-2


def test_multi_scale_frozen_plans_fit_the_arena():
    m, ts, _ = _run("1", False, [10], 6, unfreeze_after=3, multi_scale=True)
    arena = m._train_arena
    engs = [e for k, e in m._engines.items() if k[0] == "train"]
    assert engs and all(e.arena is arena for e in engs)
    assert any(not all(p.trainable) for e in engs for p in e._bwds.values())
    assert all(m._last_train_engine._bwd.trainable)


def test_freezing_everything_is_refused():
    m = build_mirror("n", nc=15, seed=0).to(DEV).train()
    with pytest.raises(RuntimeError, match="nothing is left to train"):
        TrainStep(m, batch_size=64, imgsz=128, freeze=[25])
