"""GPU tests of multi-scale training (train.py --multi-scale: TrainStep(multi_scale=True), Model.forward_train(x, size),
Model.reserve_train_arena):
  * the resize into the stem input is bit-equal to F.interpolate(bilinear, align_corners=False) + y5obb_stem_s2d, for
    down- and upscales, uint8 and fp32, square and not; sf == 1 runs today's launches;
  * plans of different shapes alias one arena: after shapes A, B, C and an arena filled with 0xFF bytes, shape A gives the
    Detect outputs and loss of a standalone plan bit for bit and its gradient within the run-to-run spread;
  * every conv / dgrad / wgrad launch of arena-built plans matches its own descriptor (tests/test_conv_plans_exact_gpu.py);
  * 20 multi-scale steps follow the fp32 CPU oracle run at the same sizes;
  * one arena, constant, for the 33 sizes of imgsz 1024; per-shape growth bounded by what the plans report; one fused
    optimizer table; run() equals the step() loop."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

from tests.lossgen import synth_targets
from tests.modelgen import build_mirror
from tests.test_conv_plans_exact_gpu import _stats, check_conv, check_wgrad
from tests.tilegen import synth_tiles
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.train_step import multi_scale_shape

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class _Sizes:
    """A generator whose draws are the given values in turn (forces the sizes a test needs)."""

    def __init__(self, values):
        self.values = list(values)

    def randrange(self, lo, hi):
        v = self.values.pop(0)
        assert lo <= v < hi
        return v


def _stem(xf):
    B, _, H, W = xf.shape
    out = torch.zeros((B, H // 2, W // 2 + 2, 16), dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().y5obb_stem_s2d(xf.contiguous().data_ptr(), out.data_ptr(), B, H, W, 1, _lib.stream_ptr()),
               "y5obb_stem_s2d")
    return out


@pytest.mark.parametrize("u8", [True, False], ids=["uint8", "fp32"])
def test_resize_into_the_stem_input_is_aten_bilinear(u8):
    from yolov5_obb_b200.train_engine import TrainEngine
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    B, S = 2, 512
    x8 = synth_tiles(B, S, seed=7).to(DEV)
    cases = [((S, S), (int(S * r), int(S * r))) for r in (0.5, 0.75, 1.0625, 1.25, 1.5)]
    cases.append(((384, 512), multi_scale_shape(512, 32, 384, 512, _Sizes([416]))[:2]))   # non-square: (320, 416)
    assert cases[-1][1] == (320, 416)
    for (H, W), (nh, nw) in cases:
        xin8 = x8[:, :, :H, :W].contiguous()
        xf = xin8.float() / torch.tensor(255.0, device=DEV)
        x = xin8 if u8 else xf
        eng = TrainEngine(m, B, nh, nw, DEV, in_hw=(H, W))
        eng.prof = {}                                # eager, with the launch kinds recorded
        with torch.no_grad():
            eng.forward(x)
        assert "resize" in eng.prof and "s2d" not in eng.prof
        want = _stem(F.interpolate(xf, size=(nh, nw), mode="bilinear", align_corners=False))
        bad = int((eng.x_s2d.view(torch.int16) != want.view(torch.int16)).sum())
        assert bad == 0, f"{H}x{W} -> {nh}x{nw}: {bad} of {want.numel()} bf16 values differ"


def test_unit_scale_step_runs_todays_launches():
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    ts = TrainStep(m, batch_size=64, imgsz=128, multi_scale=True)
    ts.rng = _Sizes([128, 96])
    imgs = synth_tiles(2, 128, seed=3).to(DEV)
    tg = torch.from_numpy(synth_targets(2, 20, 128, nc=15, seed=3)).to(DEV)
    tg0 = tg.clone()
    ts.step(imgs, tg)
    assert ts.last_shape == (128, 128)
    eng = m._last_train_engine
    assert (("train", tuple(imgs.shape), 0) in m._engines and m._engines[("train", tuple(imgs.shape), 0)] is eng
            and eng.in_hw == (eng.H, eng.W))
    eng.prof = {}
    with torch.no_grad():
        eng.forward(imgs)
    assert "s2d" in eng.prof and "resize" not in eng.prof
    ts.step(imgs, tg)
    assert ts.last_shape == (96, 96) and m._last_train_engine.in_hw == (128, 128)
    assert torch.equal(tg, tg0)                      # the caller's targets are never scaled in place


def _pass(m, x, size, tg):
    """forward_train + ComputeLoss + backward -> (Detect outputs, loss, flat gradient) copies."""
    from yolov5_obb_b200.loss import ComputeLoss
    for p in m.parameters():
        p.grad = None
    pred = m.forward_train(x, size)
    cl = getattr(m, "_test_cl", None) or ComputeLoss(m)
    m._test_cl = cl
    loss, _ = cl(pred, tg)
    outs = [p.detach().clone() for p in pred]
    loss.backward()
    g = torch.cat([p.grad.reshape(-1) for p in m.parameters()])
    return outs, loss.detach().clone(), g


def test_plans_alias_one_arena():
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n", nc=15, seed=1).train().to(DEV)
    TrainStep(m, batch_size=64, imgsz=128)                       # model.hyp / nc as training sets them
    B, S = 2, 160
    x = synth_tiles(B, S, seed=11).to(DEV)
    tg = torch.from_numpy(synth_targets(B, 30, S, nc=15, seed=11)).to(DEV)
    ref = copy.deepcopy(m)                                       # standalone plans (no arena)
    ref.hyp, ref.nc = m.hyp, m.nc
    arena = m.reserve_train_arena(B, 256, 256, DEV)
    A, Bs, C = None, (256, 256), (96, 128)
    for _ in range(2):                                           # eager, then captured graphs
        for size in (A, Bs, C):
            _pass(m, x, size, tg)
    torch.cuda.synchronize()
    arena.buf.fill_(0xFF)                                        # every arena byte NaN: stale zeros cannot survive
    arena.flat.fill_(float("nan"))
    outs, loss, g = _pass(m, x, A, tg)
    assert m._last_train_engine.arena is arena and m._last_train_engine.outside_bytes > 0
    r_outs, r_loss, g1 = _pass(ref, x, None, tg)
    _, _, g2 = _pass(ref, x, None, tg)
    assert ref._last_train_engine.arena is None
    for o, r in zip(outs, r_outs):
        assert torch.equal(o.view(torch.int32), r.view(torch.int32))
    assert torch.equal(loss.view(torch.int32), r_loss.view(torch.int32))
    assert torch.isfinite(g).all()
    spread = (g2 - g1).abs().max().item()
    err = (g - g1).abs().max().item()
    print(f"gradient: arena vs standalone {err:.3e}, standalone run-to-run spread {spread:.3e}")
    assert err <= 2.0 * spread + 1e-7 * g1.abs().max().item()


def test_every_launch_of_arena_plans_matches_its_descriptor():
    from yolov5_obb_b200.train_backward import BackwardPlan
    from yolov5_obb_b200.train_engine import TrainEngine
    torch.manual_seed(2)
    m = build_mirror("n", nc=15, seed=0).train().to(DEV)
    B, imgsz = 2, 160
    sizes = sorted({multi_scale_shape(imgsz, 32, imgsz, imgsz, _Sizes([v]))[0]
                    for v in range(int(imgsz * 0.5), int(imgsz * 1.5 + 32))}, reverse=True)
    assert sizes == [256, 224, 192, 160, 128, 96, 64]
    arena = m.reserve_train_arena(B, sizes[0], sizes[0], DEV)
    x = synth_tiles(B, imgsz, seed=1).to(DEV)
    st = _stats()
    for s in sizes:
        eng = TrainEngine(m, B, s, s, DEV, in_hw=(imgsz, imgsz), arena=arena)
        with torch.no_grad():
            eng.forward(x)                                       # the plan uses the arena after the larger one did
        plan = BackwardPlan(eng)
        convs = [lay.conv for lay in eng.conv_layers] + list(eng.det_convs)
        wgrads = []
        for part in plan.det_parts + plan.conv_parts:
            convs += part.get("dgrad_ops", [])
            wgrads.append(part["wgrad"])
        for i, op in enumerate(convs):
            check_conv(op, st, f"{s}x{s} conv {i}")
        for i, wg in enumerate(wgrads):
            check_wgrad(wg, st, f"{s}x{s} wgrad {i}")
        del plan, eng
    print(f"\n{len(sizes)} arena plans: {st['conv']} conv and {st['wgrad']} wgrad launches checked, {st['bitwise']} bitwise")
    assert st["conv"] > 0 and st["wgrad"] > 0


def _oracle_multiscale(m, imgs_u8, tg, shapes, imgsz, emulate_bf16):
    """train.py:296-342 with --multi-scale on the CPU in fp32 (oracle/model_ref + loss_ref + torch.optim.SGD), the sizes given:
    F.interpolate of the batch and targets[:, 2:6] * label_ratio, as train.py:317-320."""
    from oracle import loss_ref, model_ref
    from yolov5_obb_b200.train_step import HYP_FINETUNE_DOTA, param_groups
    m = copy.deepcopy(m).cpu().train()
    det = m.model[-1]
    hyp = loss_ref.scaled_hyp({k: HYP_FINETUNE_DOTA.get(k, v) for k, v in loss_ref.DEFAULT_HYP.items()}, det.nl, det.nc, imgsz)
    g0, g1, g2 = param_groups(m)
    opt = torch.optim.SGD(g0, lr=HYP_FINETUNE_DOTA["lr0"], momentum=HYP_FINETUNE_DOTA["momentum"], nesterov=True)
    opt.add_param_group({"params": g1, "weight_decay": HYP_FINETUNE_DOTA["weight_decay"]})
    opt.add_param_group({"params": g2})
    x0 = imgs_u8.float().cpu() / 255
    out = []
    for ns in shapes:
        x, t = x0, tg.cpu().clone()
        if tuple(ns) != tuple(x0.shape[2:]):
            x = F.interpolate(x0, size=list(ns), mode="bilinear", align_corners=False)
            t[:, 2:6] *= float(ns[0]) / x0.shape[2]
        with torch.enable_grad():
            pred = model_ref.forward_with_grad(m, x, training=True, emulate_bf16=emulate_bf16)
            loss, _ = loss_ref.compute_loss(pred, t, det.anchors, det.stride, hyp, det.nc)
            loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        out.append(loss.item())
    return out


def test_multiscale_loss_trajectory_against_the_cpu_oracle():
    """The criterion of test_train_step_gpu.test_loss_trajectory_against_the_cpu_oracle, over 20 multi-scale steps."""
    from yolov5_obb_b200.train_step import TrainStep
    B, S, N = 4, 128, 20
    m0 = build_mirror("n", nc=15, seed=1).train()
    imgs = synth_tiles(B, S, seed=3)
    tg = torch.from_numpy(synth_targets(B, 40, S, nc=15, seed=3))
    md = copy.deepcopy(m0).to(DEV)
    ts = TrainStep(md, batch_size=64, imgsz=S, multi_scale=True, seed=3)
    dev, shapes = [], []
    xd, td = imgs.to(DEV), tg.to(DEV)
    for _ in range(N):
        l, _ = ts.step(xd, td)
        dev.append(l.item())
        shapes.append(ts.last_shape)
    assert len(set(shapes)) >= 3, shapes
    ref = _oracle_multiscale(m0, imgs, tg, shapes, S, emulate_bf16=False)
    emu = _oracle_multiscale(m0, imgs, tg, shapes, S, emulate_bf16=True)
    print("sizes       ", [s[0] for s in shapes])
    print("oracle fp32 ", [f"{v:.3f}" for v in ref])
    print("oracle bf16 ", [f"{v:.3f}" for v in emu])
    print("device      ", [f"{v:.3f}" for v in dev])
    assert abs(dev[0] - ref[0]) < 1e-3 * abs(ref[0]) + 2e-2 * abs(emu[0] - ref[0]) + 1e-3
    run_max = 0.0
    for i in range(N):
        run_max = max(run_max, abs(emu[i] - ref[i]))
        assert abs(dev[i] - ref[i]) < 3.0 * run_max + 0.02 * abs(ref[i]) + 1e-3, (i, shapes[i], dev[i], ref[i], emu[i])


def test_one_arena_for_the_33_sizes_of_imgsz_1024():
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("s", nc=15, seed=1).train().to(DEV)
    B, S = 16, 1024
    ts = TrainStep(m, batch_size=B, imgsz=S, multi_scale=True)
    arena = m._train_arena
    ptr = arena.buf.data_ptr()
    imgs = synth_tiles(B, S, seed=5).to(DEV)
    tg = torch.from_numpy(synth_targets(B, 200, S, nc=15, seed=5)).to(DEV)
    draws = list(range(512, 1537, 32))
    ts.rng = _Sizes(draws + draws)
    ts.step(imgs, tg)                                            # 512: the allocator's and the loss's first-use state settle
    torch.cuda.synchronize()
    mem0 = torch.cuda.memory_allocated()
    seen = [ts.last_shape]
    for _ in draws[1:]:
        ts.step(imgs, tg)
        seen.append(ts.last_shape)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - mem0
    engines = [e for k, e in m._engines.items() if k[0] == "train"]
    assert sorted(s[0] for s in seen) == list(range(512, 1537, 32)) and len(engines) == 33
    assert all(e.arena is arena for e in engines) and m._train_arena is arena and arena.buf.data_ptr() == ptr
    outside = {e.H: e.outside_bytes for e in engines}
    first = [e for e in engines if e.H == 512][0]
    bound = sum(v for h, v in outside.items() if h != 512)
    print(f"\narena {arena.nbytes / 2**30:.2f} GiB; growth over 32 new sizes {grown / 2**20:.1f} MiB; reported outside "
          f"the arena {bound / 2**20:.1f} MiB (largest plan {max(outside.values()) / 2**20:.1f} MiB)")
    assert grown <= bound + 64 * 2**20
    assert max(outside.values()) * 33 < arena.nbytes                # the per-shape cost is small beside the arena
    assert first.outside_bytes > 0
    for _ in range(3):                                           # second visits reuse the plans and the arena
        ts.step(imgs, tg)
    assert len([k for k in m._engines if k[0] == "train"]) == 33 and arena.buf.data_ptr() == ptr


def test_run_equals_the_step_loop():
    from yolov5_obb_b200.train_step import TrainStep
    B, S = 2, 128
    batches = [(synth_tiles(B, S, seed=10 + i).pin_memory(),
                torch.from_numpy(synth_targets(B, 10 + 7 * i, S, nc=15, seed=20 + i)).pin_memory()) for i in range(6)]
    ma = build_mirror("n", nc=15, seed=4).train().to(DEV)
    mb = copy.deepcopy(ma)
    ta = TrainStep(ma, batch_size=64, imgsz=S, multi_scale=True, seed=9)
    tb = TrainStep(mb, batch_size=64, imgsz=S, multi_scale=True, seed=9)
    want, sa, fused = [], [], []
    for x, t in batches:
        l, _ = ta.step(x.to(DEV), t.to(DEV))
        want.append(l.item())
        sa.append(ta.last_shape)
        fused.append(ta._fused)
    assert fused[0] is not None and all(f is fused[0] for f in fused)   # the fused optimizer table is built once
    sb, step = [], tb.step

    def recording(*a):
        r = step(*a)
        sb.append(tb.last_shape)
        return r
    tb.step = recording
    got = [l.item() for l, _ in tb.run(iter(batches))]
    assert sb == sa and len(set(sa)) > 1, (sa, sb)
    assert abs(got[0] - want[0]) <= 1e-5 * max(1.0, abs(want[0]))
    assert all(math.isfinite(v) for v in got)
