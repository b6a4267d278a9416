"""The four-level P6 family (models/hub/yolov5{n,s,m,l,x}6.yaml: stride 64, a fourth Detect level) through every device entry
point: eval and records, the loss at nl = 4, training (SGD / Adam, fused / torch, multi-scale with gs = 64), the validation loss,
TTA, whole scenes at 1088^2 and images of any size.  The yardsticks are those of the P5 tests, imported rather than restated:
test_engine_gpu's tolerance, test_loss_gpu's golden tolerances, tests/lossref.py's fp64 bounds, test_train_backward_gpu's
teacher forcing, test_train_step_gpu's oracle trajectory, test_valloss_gpu's exact-logit head, test_conv_plans_exact_gpu's
integer-operand launch checks."""
import copy
import gc
import types
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref, scene_ref, tta_ref
from tests import lossref, p6gen
from tests import test_conv_plans_exact_gpu as CE
from tests import test_scene_gpu as SC
from tests import test_valloss_gpu as VL
from tests.lossgen import synth_targets
from tests.modelgen import build_mirror, calibrated_bench_model
from tests.recordcheck import check_records
from tests.test_engine_gpu import _compare
from tests.test_train_backward_gpu import _teacher_forced
from tests.test_train_step_gpu import _oracle_trajectory
from tests.tilegen import synth_tiles
from tests.ttagen import pieces
from yolov5_obb_b200 import general
from yolov5_obb_b200 import yolo as Y
from yolov5_obb_b200.loss import ComputeLoss
from yolov5_obb_b200.scene import SceneDetector, split_origins

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
DEV = "cuda:0"
G = np.load(ROOT / "tests" / "golden" / "p6_golden.npz")
P6_CHANNELS = {"n": (64, 128, 192, 256), "s": (128, 256, 384, 512)}


class FakeP6Model:
    """What ComputeLoss reads from a model (.hyp, .model[-1]) for the P6 Detect."""

    def __init__(self, hyp, nc=15):
        self.hyp = hyp
        det = Y.Detect(nc=nc, anchors=p6gen._ANCH.view(4, -1).tolist(), ch=(8,) * 4)
        det.stride = torch.tensor(p6gen.STRIDES)
        det.anchors /= det.stride.view(-1, 1, 1)
        self.model = [det]


def _release_memory():
    """Plans of earlier tests (and their launch closures' reference cycles) hold device memory the large plans here need."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _golden_hyp():
    v = G["loss/hyp"]
    return dict(loss_ref.DEFAULT_HYP, box=float(v[0]), obj=float(v[1]), cls=float(v[2]), theta=float(v[3]),
                anchor_t=float(v[4]), label_smoothing=0.0)


def _compare_pieces(got, key, what):
    _compare(torch.from_numpy(got["rows"]), torch.from_numpy(G[f"{key}/rows"]), f"{what} sampled rows")
    box, ref = torch.from_numpy(got["box"]), torch.from_numpy(G[f"{key}/box"])
    frac_bad = ((box - ref).abs() > ref.abs() * 3e-2 + 3e-2).float().mean().item()
    print(f"{what} boxes: max err {(box - ref).abs().max().item():.4g}, out-of-tol {frac_bad:.2e}")
    assert frac_bad < 1e-3


# ---- inference -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", ["n6", "s6"])
def test_eval_and_tta_match_reference_golden(size):
    m = build_mirror(size, nc=15, seed=0)
    md = copy.deepcopy(m).to(DEV)
    x = p6gen.eval_input()
    pred, _ = md(x.to(DEV))
    assert pred.shape == (1, 1530, 200)
    _compare_pieces(pieces(pred.cpu().numpy()), f"{size}/eval", f"yolov5{size} eval vs golden")
    ref, _ = model_ref.forward(m, x)
    _compare(pred, ref, f"yolov5{size} eval vs fp32 oracle")
    xt = p6gen.tta_input()
    aug, none = md.forward_augment(xt.to(DEV))
    assert none is None and tuple(aug.shape) == tuple(G[f"{size}/tta/shape"])
    _compare_pieces(pieces(aug.cpu().numpy()), f"{size}/tta", f"yolov5{size} TTA vs golden")
    want, _ = tta_ref.forward_augment(m, xt)
    _compare(aug, want, f"yolov5{size} TTA vs fp32 oracle")


def test_yolov5s6_b16_1280_plan_matches_oracle():
    """The 1280^2 batch-16 plan (20 x 20 P6 maps) against the fp32 oracle on two sampled images, with bench.parity_gate's
    measured bf16 yardstick, on the calibrated model the benchmark uses."""
    import bench
    m_cpu = calibrated_bench_model("s6", nc=15, seed=0)
    m = copy.deepcopy(m_cpu).to(DEV)
    x = synth_tiles(16, 1280, seed=0).to(DEV)
    pred, _ = m(x)
    torch.cuda.synchronize()
    assert pred.shape == (16, 3 * (160 ** 2 + 80 ** 2 + 40 ** 2 + 20 ** 2), 200)
    out = bench.parity_gate(m_cpu, x, pred, sample=(0, -1))
    print(out)
    assert out["ok"] and len(out["levels"]) == 4


@pytest.mark.parametrize("augment", [False, True], ids=["plain", "tta"])
def test_records_plus_nms_equal_tensor_plus_nms(augment):
    m = build_mirror("s6", nc=15, seed=3, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    x = torch.rand(2, 3, 256, 320, generator=torch.Generator().manual_seed(2)).to(DEV)
    pred = (m.forward_augment(x) if augment else m(x))[0].clone()
    rec = m.detect_records(x, augment=augment)
    pred, near_ties = check_records(pred, rec.data, 15)
    assert near_ties <= max(2, pred.shape[0] * pred.shape[1] // 1000)
    for kw in (dict(multi_label=True, max_det=300), dict(multi_label=False, max_det=100)):
        a = general.non_max_suppression_obb(pred, 0.25, 0.45, **kw)
        b = general.non_max_suppression_obb(rec, 0.25, 0.45, **kw)
        assert sum(t.shape[0] for t in a) > 0
        for u, v in zip(a, b):
            assert torch.equal(u, v)


# ---- loss ------------------------------------------------------------------------------------------------------------
def test_loss_matches_reference_golden():
    cl = ComputeLoss(FakeP6Model(_golden_hyp()))
    p = [x.to(DEV).requires_grad_(True) for x in p6gen.loss_preds(seed=7)]
    tg = torch.from_numpy(G["loss/targets"]).to(DEV)
    loss, items = cl(p, tg)
    np.testing.assert_allclose(loss.detach().cpu().numpy(), G["loss/loss"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(items.cpu().numpy(), G["loss/items"], rtol=0, atol=1e-4)
    (loss * 3.0).backward()
    for i, x in enumerate(p):
        g = x.grad.reshape(-1, 200).cpu()
        np.testing.assert_allclose(g[:, 4].numpy(), G[f"loss/gobj{i}"], rtol=2e-5, atol=1e-7)
        rows = G[f"loss/grows{i}"]
        assert rows.size > 0
        np.testing.assert_allclose(g[rows].numpy(), G[f"loss/gvals{i}"], rtol=2e-4, atol=2e-7)
        rest = g.clone()
        rest[:, 4] = 0
        rest[rows] = 0
        assert rest.abs().max().item() == 0.0


@pytest.mark.parametrize("cols", [187, 8, 7])
def test_loss_element_by_element_against_fp64(cols, monkeypatch):
    """tests/lossref.py's per-element bounds with the four-level balance; the large targets match on P6 only."""
    from tests.lossgen import compact_layouts
    monkeypatch.setattr(lossref, "BALANCE", (4.0, 1.0, 0.25, 0.06))
    hyp = _golden_hyp()
    p = p6gen.loss_preds(seed=3)
    tg = compact_layouts(p6gen.loss_targets(seed=3))[cols]
    cl = ComputeLoss(FakeP6Model(hyp))
    anchors, strides = p6gen.ANCHORS_GRID, p6gen.STRIDES
    ref = lossref.reference(p, tg, hyp, 15, anchors, strides)
    bnd = lossref.bounds(p, tg, hyp, 15, anchors, strides)
    assert all(n > 0 for n in bnd["nrows"]), bnd["nrows"]
    pd = [x.to(DEV).requires_grad_(True) for x in p]
    loss, items = cl(pd, tg.to(DEV))
    worst = {}
    for gl in (1.0, 2.0 ** 16):
        grads = torch.autograd.grad(loss, pd, torch.full_like(loss, gl), retain_graph=True)
        for k, v in lossref.check(grads, loss, items, ref, bnd, gl).items():
            worst[k] = max(worst.get(k, 0.0), v)
    print(f"\nP6 {cols} columns: rows per level {bnd['nrows']}; worst error / bound: "
          + ", ".join(f"{k} {v:.3g}" for k, v in sorted(worst.items())))


def test_head_items_bit_equal_to_loss_on_materialised_logits(monkeypatch):
    """The validation loss from the Detect inputs against ComputeLoss on the materialised head output, with exact logits
    (test_valloss_gpu's integer head, four levels): loss and items bit for bit."""
    monkeypatch.setattr(VL, "STRIDES", tuple(int(s) for s in p6gen.STRIDES))
    B, H, W = 2, 256, 320
    cl = ComputeLoss(FakeP6Model(loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 4, 15, W)))
    levels, ps = VL._integer_head(B, H, W, P6_CHANNELS["s"], seed=4)
    tg = torch.from_numpy(p6gen.p6_targets(B, H, W, seed=4)).to(DEV)
    rc, loss, items, _ = VL._forward_head(cl, levels, tg, B)
    assert rc == 0
    want_loss, want_items = cl(ps, tg)
    assert torch.equal(loss, want_loss.detach()) and torch.equal(items, want_items), (items, want_items)


def test_validator_plan_head_items_match_oracle():
    """head_items over the four levels a records plan keeps, against the fp32 oracle's loss on the plan's own features."""
    m = build_mirror("s6", nc=15, seed=0, obj_bias=-2.0).to(DEV)
    m.hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 4, 15, 320)
    cl = ComputeLoss(m)
    im = torch.rand(2, 3, 256, 320, generator=torch.Generator().manual_seed(5))
    tg = torch.from_numpy(p6gen.p6_targets(2, 256, 320, seed=5))
    m.detect_records(im.to(DEV))
    plan = m.records_plan(tuple(im.shape), DEV)
    loss, items = cl.head_items(plan, tg.to(DEV))
    det = copy.deepcopy(m.model[-1]).cpu()
    feats = []
    for l, (x, w, b) in enumerate(plan.head_inputs()):
        feats.append(x.view().permute(0, 3, 1, 2).float().cpu())
        with torch.no_grad():
            det.m[l].weight.copy_(w.float().cpu().view_as(det.m[l].weight))
            det.m[l].bias.copy_(b.cpu())
    assert len(feats) == 4
    raw = model_ref.detect_fwd(det, feats, training=True)
    want_loss, want_items = loss_ref.compute_loss(raw, tg, det.anchors, det.stride, m.hyp, 15)
    np.testing.assert_allclose(items.cpu().numpy(), want_items.numpy(), rtol=1e-5, atol=0)
    np.testing.assert_allclose(loss.cpu().numpy(), want_loss.detach().numpy(), rtol=1e-5, atol=0)


# ---- training --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(1, 128, 192), (2, 256, 320)])
def test_train_forward_matches_oracle(B, H, W):
    """Batch-statistic BatchNorm amplifies storage rounding layer by layer, and the P6 maps normalise over a handful of
    pixels: test_train_forward_gpu's rule, per Detect level the relative L2 distance to the fp32 oracle below 1.5x that of the
    bf16-emulating oracle + 3e-3.  At 1 x 128 x 192 the fp32 oracle is the one test_p6_cpu pins to the reference golden."""
    m = build_mirror("s6", nc=15, seed=0).train()
    x = p6gen.eval_input() if B == 1 else torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(9))
    want = model_ref.forward(copy.deepcopy(m), x, training=True)
    emu = model_ref.forward(copy.deepcopy(m), x, training=True, emulate_bf16=True)
    with torch.no_grad():
        raw = m.to(DEV)(x.to(DEV))
    assert len(raw) == 4
    for i, (r, w, e) in enumerate(zip(raw, want, emu)):
        assert r.shape == w.shape
        rel = ((r.cpu() - w).norm() / w.norm()).item()
        floor = ((e - w).norm() / w.norm()).item()
        print(f"level {i}: rel L2 {rel:.3g}, bf16 floor {floor:.3g}")
        assert rel < 1.5 * floor + 3e-3, (i, rel, floor)


@pytest.mark.parametrize("size,B,H,W", [("n6", 2, 256, 320), ("s6", 2, 256, 256)])
def test_backward_teacher_forced_parity(size, B, H, W):
    """test_train_backward_gpu's one-module-deep teacher forcing, on the P6 graph (tolerances of that test)."""
    m = build_mirror(size, nc=15, seed=3).train()
    ref_m = copy.deepcopy(m)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(B, 3, H, W, generator=g)
    md = m.to(DEV)
    outs = md(x.to(DEV))
    assert len(outs) == 4
    Gr = [torch.randn(o.shape, generator=g) * 0.05 for o in outs]
    sum((o * gg.to(DEV)).sum() for o, gg in zip(outs, Gr)).backward()
    torch.cuda.synchronize()
    eng = [e for k, e in md._engines.items() if k[0] == "train"][0]
    pg, gl, gout, inner = _teacher_forced(md, ref_m, eng, x, Gr)
    rels, bad = [], []
    for n, p in md.named_parameters():
        rel = (p.grad.float().cpu() - pg[n]).norm().item() / max(pg[n].norm().item(), 1e-12)
        rels.append(rel)
        if rel >= 6e-2:
            bad.append((n, rel))
    rels.sort()
    print(f"{size}: {len(rels)} parameter tensors: median rel {rels[len(rels) // 2]:.3g}, max {rels[-1]:.3g}")
    assert not bad, bad[:10]
    assert rels[len(rels) // 2] < 2e-2
    grels = [((gout(i) - ref).norm().item() / max(ref.norm().item(), 1e-12), i) for i, ref in sorted(gl.items())]
    assert max(r for r, _ in grels) < 6e-2, grels
    for i, (want, have) in inner.items():
        assert (have - want).norm().item() / max(want.norm().item(), 1e-12) < 3e-2


def _adam_oracle_trajectory(m, imgs_u8, tg, steps, imgsz, emulate_bf16):
    """_oracle_trajectory with train.py --adam: torch.optim.Adam(g0, lr0, betas=(momentum, 0.999)) and the same groups."""
    from yolov5_obb_b200.train_step import HYP_FINETUNE_DOTA, param_groups
    m = copy.deepcopy(m).cpu().train()
    det = m.model[-1]
    hyp = loss_ref.scaled_hyp({k: HYP_FINETUNE_DOTA.get(k, v) for k, v in loss_ref.DEFAULT_HYP.items()}, det.nl, det.nc, imgsz)
    g0, g1, g2 = param_groups(m)
    opt = torch.optim.Adam(g0, lr=HYP_FINETUNE_DOTA["lr0"], betas=(HYP_FINETUNE_DOTA["momentum"], 0.999))
    opt.add_param_group({"params": g1, "weight_decay": HYP_FINETUNE_DOTA["weight_decay"]})
    opt.add_param_group({"params": g2})
    x = imgs_u8.float().cpu() / 255
    out = []
    for _ in range(steps):
        with torch.enable_grad():
            pred = model_ref.forward_with_grad(m, x, training=True, emulate_bf16=emulate_bf16)
            loss, _ = loss_ref.compute_loss(pred, tg.cpu(), det.anchors, det.stride, hyp, det.nc)
            loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
        out.append(loss.item())
    return out


@pytest.mark.parametrize("adam,fused", [(False, "1"), (False, "0"), (True, "1"), (True, "0")],
                         ids=["sgd-fused", "sgd-torch", "adam-fused", "adam-torch"])
def test_loss_trajectory_against_the_cpu_oracle(adam, fused, monkeypatch):
    """test_train_step_gpu's yardstick over 8 steps of yolov5n6 at 128 x 192 on one repeated batch: step 0 to 1e-3, then within
    3x the bf16-emulating oracle's own drift + 2 % of the loss."""
    from yolov5_obb_b200.train_step import TrainStep
    monkeypatch.setenv("Y5OBB_FUSED_SGD", fused)
    B, H, W, N = 2, 128, 192, 8
    m0 = build_mirror("n6", nc=15, seed=1).train()
    imgs = torch.cat([synth_tiles(B, W, seed=3)[:, :, :H]], 0).contiguous()
    tg = torch.from_numpy(p6gen.p6_targets(B, H, W, nt=30, seed=3))
    traj = _adam_oracle_trajectory if adam else _oracle_trajectory
    ref = traj(m0, imgs, tg, N, W, emulate_bf16=False)
    emu = traj(m0, imgs, tg, N, W, emulate_bf16=True)
    md = copy.deepcopy(m0).to(DEV)
    ts = TrainStep(md, batch_size=64, imgsz=W, adam=adam)
    assert ts._use_fused == (fused == "1") and ts.gs == 64
    dev = []
    for _ in range(N):
        l, _ = ts.step(imgs.to(DEV), tg.to(DEV))
        dev.append(l.item())
    print("oracle fp32 ", [f"{v:.3f}" for v in ref])
    print("oracle bf16 ", [f"{v:.3f}" for v in emu])
    print("device      ", [f"{v:.3f}" for v in dev])
    assert abs(dev[0] - ref[0]) < 1e-3 * abs(ref[0]) + 2e-2 * abs(emu[0] - ref[0]) + 1e-3
    run_max = 0.0
    for i in range(N):
        run_max = max(run_max, abs(emu[i] - ref[i]))
        assert abs(dev[i] - ref[i]) < 3.0 * run_max + 0.02 * abs(ref[i]) + 1e-3, (i, dev[i], ref[i], emu[i])


def test_multi_scale_steps_at_512_and_1536_from_one_arena():
    """TrainStep(multi_scale=True) with gs = 64 reserves one arena for 1536^2 at imgsz 1024; steps drawn at 512^2 and 1536^2
    run from it, and each equals a standalone plan of that size on the same resized batch (same forward bits, same loss)."""
    from tests.test_multiscale_gpu import _pass
    from yolov5_obb_b200.train_step import TrainStep
    _release_memory()
    B = 2
    m = build_mirror("n6", nc=15, seed=1).train().to(DEV)
    ts = TrainStep(m, batch_size=B, imgsz=1024, multi_scale=True)   # the arena is sized for batch_size images of 1536^2
    assert ts.gs == 64 and m._train_arena is not None
    x = synth_tiles(B, 1024, seed=11).to(DEV)
    tg = torch.from_numpy(synth_targets(B, 30, 1024, nc=15, seed=11)).to(DEV)
    ref = copy.deepcopy(m)
    ref.hyp, ref.nc = m.hyp, m.nc
    for S in (512, 1536):
        outs, loss, g = _pass(m, x, (S, S), tg)
        assert m._last_train_engine.arena is m._train_arena
        r_outs, r_loss, _ = _pass(ref, x, (S, S), tg)
        assert ref._last_train_engine.arena is None
        assert [tuple(o.shape[2:4]) for o in outs] == [(S // s, S // s) for s in (8, 16, 32, 64)]
        for o, r in zip(outs, r_outs):
            assert torch.equal(o.view(torch.int32), r.view(torch.int32))
        assert torch.equal(loss.view(torch.int32), r_loss.view(torch.int32))
        assert torch.isfinite(g).all()
    for S in (512, 1536):     # and through TrainStep's own draw
        ts.rng = type("Fixed", (), {"randrange": staticmethod(lambda lo, hi, v=S: v)})()
        l, _ = ts.step(x, tg)
        assert ts.last_shape == (S, S) and torch.isfinite(l).all()


# ---- whole scenes and images of any size -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene_model():
    return build_mirror("n6", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)


def test_scene_detector_equals_composed_public_calls_at_1088(scene_model):
    """val.py's rect pad 0.5 with the model stride 64: 1088^2 tiles, border 32."""
    scene = SC._scene(1700, 2300, 2)
    det = SceneDetector(scene_model, batch_size=4)
    assert (det.size, det.border, det.pad_xy) == (1088, 32, 32.0)
    _release_memory()
    origins = split_origins(*scene.shape[:2])
    tiles = SC._torch_tiles(scene, origins, 1024, 1088, 32).to(DEV)
    dets = []
    for t0 in range(0, len(origins), 4):    # the public calls, four tiles at a time as the detector runs them
        dets += general.non_max_suppression_obb(scene_model(tiles[t0:t0 + 4].contiguous())[0], 0.01, 0.4, multi_label=True,
                                                max_det=1500)
    rows = torch.zeros((len(origins), 1500, 7), device=DEV)
    counts = torch.tensor([d.shape[0] for d in dets], device=DEV)
    for t, d in enumerate(dets):
        rows[t, :d.shape[0]] = d
    tl = [(l, u) + d for (l, u), d in zip(origins, SC._device_polys(rows, counts, 32.0))]
    want = torch.from_numpy(scene_ref.merge(tl, 15, 0.2))
    got = det.det(scene.to(DEV)).rows.cpu()
    assert int(counts.sum()) > 1000 and want.shape[0] > 100
    assert torch.equal(got, want)


def test_scene_detector_tile_size_follows_the_model_stride(scene_model):
    """The tile size is rounded to the model's largest stride, as the reference's rect loader does: 1088^2 for the P6 strides
    (8, 16, 32, 64), 1056^2 for P5 at pad 0.5; stride sets of neither family are refused."""
    assert SceneDetector(scene_model).size == 1088
    for strides, size in (([8.0, 16.0, 32.0, 64.0], 1088), ([8.0, 16.0, 32.0], 1056)):
        det = SceneDetector(types.SimpleNamespace(stride=torch.tensor(strides)))
        assert (det.size, det.border, det.pad_xy) == (size, (size - 1024) // 2, (size - 1024) / 2)
    for strides in ([8.0, 16.0, 64.0], [8.0, 16.0, 32.0, 64.0, 128.0], [16.0, 32.0, 64.0]):
        with pytest.raises(RuntimeError, match="stride"):
            SceneDetector(types.SimpleNamespace(stride=torch.tensor(strides)))


def test_run_images_defaults_to_the_model_stride(scene_model):
    """detect.py's letterbox to the minimum rectangle, rounded to the model's stride (64) when none is given."""
    from yolov5_obb_b200.pipeline import DetectPipeline
    rng = np.random.default_rng(0)
    images = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((300, 500), (640, 200), (384, 384))]
    pipe = DetectPipeline(scene_model, conf_thres=0.25, iou_thres=0.45, multi_label=True, device=DEV, slots=1)
    got = list(pipe.run_images(images, img_size=640))
    want = list(pipe.run_images(images, img_size=640, stride=64))
    assert len(got) == 3
    for a, b in zip(got, want):
        assert a.shapes == b.shapes and torch.equal(a.rows, b.rows)
    with pytest.raises(RuntimeError, match="multiple of the model's largest stride"):
        list(pipe.run_images(images, img_size=640, stride=32))


def test_augment_loader_at_a_multiple_of_64():
    """DeviceAugmentLoader at imgsz 192 (a multiple of 64): its batch feeds a P6 TrainStep."""
    from tests.augmentgen import HYP_DOTA, synth_dataset
    from yolov5_obb_b200.augment import DeviceAugmentLoader, DeviceDataset
    from yolov5_obb_b200.train_step import TrainStep
    images, labels = synth_dataset(6, 192, 9)
    loader = DeviceAugmentLoader(DeviceDataset(images, labels, 192, DEV), dict(HYP_DOTA), batch_size=2, shuffle=True, seed=5)
    imgs, tg = next(iter(loader))
    assert imgs.shape[2:] == (192, 192) and tg.shape[0] > 0
    m = build_mirror("n6", nc=15, seed=1).train().to(DEV)
    ts = TrainStep(m, batch_size=2, imgsz=192)
    l, items = ts.step(imgs, tg)
    assert torch.isfinite(l).all() and torch.isfinite(items).all()


# ---- every conv / dgrad / wgrad launch, exact under integer operands -------------------------------------------------
@pytest.mark.parametrize("size,B,H,W,kind", [("s6", 16, 1280, 1280, "forward"), ("s6", 8, 1024, 1024, "train")],
                         ids=["yolov5s6-b16-1280-forward", "yolov5s6-b8-1024-train"])
def test_every_launch_matches_its_descriptor(size, B, H, W, kind, monkeypatch):
    _release_memory()
    CE.test_every_launch_matches_its_descriptor(size, B, H, W, kind, None, monkeypatch)
