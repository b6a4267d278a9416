"""GPU tests of test-time augmentation (Model.forward_augment, detect_records(augment=True), Validator(augment=True),
engine.TTAPlan, y5obb_scale_img_s2d, the Detect epilogue's de-scale):
  * the resample is bit-equal to ATen's F.interpolate / F.pad composition put through the stem layout pass;
  * each branch's rows equal the plain engine's forward of the composed input, de-scaled with ATen ops and clipped
    (_forward_augment restated around the engine's own forward) - branch 0 equals the plain forward itself;
  * the whole output against the REFERENCE model's golden and, at the benchmarked shape, against the fp32 oracle;
  * records + NMS equal tensor + NMS; the Validator equals the composition of the public calls;
  * the pruned plans, the re-plan after a parameter update, and the refusals."""
import copy
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref, tta_ref
from tests.modelgen import build_mirror
from tests.recordcheck import check_records
from tests.test_engine_gpu import _compare
from tests.ttagen import pieces, tta_input
from yolov5_obb_b200 import _lib, general
from yolov5_obb_b200.engine import TTA_PAD, tta_geometry

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
DEV = "cuda:0"


def _composed(x, g):
    """scale_img(x.flip(3) if flipped else x) with ATen's own ops on the device (x fp32)."""
    xi = x.flip(3) if g["flip"] == 3 else x
    xi = F.interpolate(xi, size=(g["h"], g["w"]), mode="bilinear", align_corners=False)
    return F.pad(xi, [0, g["Wp"] - g["w"], 0, g["Hp"] - g["h"]], value=TTA_PAD)


def _stem(xf):
    B, _, H, W = xf.shape
    out = torch.zeros((B, H // 2, W // 2 + 2, 16), dtype=torch.bfloat16, device=DEV)
    _lib.check(_lib.lib().y5obb_stem_s2d(xf.contiguous().data_ptr(), out.data_ptr(), B, H, W, 1, _lib.stream_ptr()),
               "y5obb_stem_s2d")
    return out


def _descaled(pred, g, W):
    p = pred.clone()
    if g["scale"] != 1:
        p[..., :4] /= g["scale"]
        if g["flip"] == 3:
            p[..., 0] = W - p[..., 0]
    starts = np.cumsum([0] + g["level_rows"])
    return torch.cat([p[:, int(starts[l]):int(starts[l + 1])] for l in g["levels"]], 1)


@pytest.fixture(scope="module")
def model_n():
    return build_mirror("n", nc=15, seed=1).to(DEV)


@pytest.mark.parametrize("B,H,W", [(1, 64, 64), (3, 128, 160), (1, 608, 1024), (3, 1024, 1024)])
def test_resample_equals_aten_composition(model_n, B, H, W):
    g = torch.Generator().manual_seed(H + W + B)
    u8 = torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    xf = torch.rand(B, 3, H, W, generator=g).to(DEV)
    plan = model_n.tta_plan((B, 3, H, W), DEV)
    for x, xa in ((xf, xf), (u8, u8.float() / torch.tensor(255.0, device=DEV))):
        plan.forward(x)
        for k in (1, 2):
            want = _stem(_composed(xa, plan.branches[k]))
            assert torch.equal(plan.engines[k].x_s2d, want), (x.dtype, k)


def test_branches_equal_plain_forward_of_composed_input(model_n):
    B, H, W = 2, 1024, 1024
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(7)).to(DEV)
    pred = model_n.forward_augment(x)[0].clone()
    recs = model_n.detect_records(x, augment=True).data.clone()
    branches, rows = tta_geometry(H, W)
    assert pred.shape == (B, rows, 200) and rows == 114627
    # branch 0: the plain forward's first two levels, bit for bit (tensor and records)
    r0 = branches[0]["rows"]
    assert r0 == 61440
    assert torch.equal(pred[:, :r0], model_n(x)[0][:, :r0])
    assert torch.equal(recs[:, :r0], model_n.detect_records(x).data[:, :r0])
    # branches 1, 2: the plain engine on ATen's composed input, de-scaled with ATen ops, clipped
    for g in branches[1:]:
        want = _descaled(model_n(_composed(x, g))[0], g, W)
        assert torch.equal(pred[:, g["row_off"]:g["row_off"] + g["rows"]], want), g["scale"]
        # the records' box / obj / class columns are the same de-scaled values
        assert torch.equal(recs[:, g["row_off"]:g["row_off"] + g["rows"], :20], want[..., :20]), g["scale"]


@pytest.mark.parametrize("size", ["n", "s"])
def test_forward_augment_matches_reference_golden(size):
    """Every row's box columns and every column of the sampled rows (tests/ttagen.py) with test_engine_gpu._compare's
    tolerance: 3e-2 relative + absolute, under 1e-3 of the elements out."""
    G = np.load(ROOT / "tests" / "golden" / "tta_golden.npz")
    m = build_mirror(size, nc=15, seed=0).to(DEV)
    x = tta_input()
    assert x.double().sum().item() == float(G["x_sum"])
    pred, none = m.forward_augment(x.to(DEV))
    torch.cuda.synchronize()
    assert none is None and tuple(pred.shape) == tuple(G[f"{size}/shape"]) == (2, 2640, 200)
    got = pieces(pred.cpu().numpy())
    _compare(torch.from_numpy(got["rows"]), torch.from_numpy(G[f"{size}/rows"]), f"yolov5{size} TTA sampled rows vs golden")
    box, ref = torch.from_numpy(got["box"]), torch.from_numpy(G[f"{size}/box"])
    frac_bad = ((box - ref).abs() > ref.abs() * 3e-2 + 3e-2).float().mean().item()
    print(f"yolov5{size} TTA boxes vs golden: max err {(box - ref).abs().max().item():.4g}, out-of-tol {frac_bad:.2e}")
    assert frac_bad < 1e-3


def test_bench_shape_yolov5s_b16_1024_matches_oracle():
    """yolov5s b16 x 1024^2, uint8 input, against the fp32 oracle's forward_augment on two sampled images, with the criterion of
    test_engine_gpu.test_bench_plan_yolov5s_b16_1024_matches_oracle (bench.parity_gate) applied per branch and level: relative
    L2 < 2 x the bf16-storage floor + 3e-3, and the `obj > conf` candidate masks agree no worse than the floor's - 0.1."""
    import bench
    m_cpu = bench.build_model("s")
    m = copy.deepcopy(m_cpu).to(DEV)
    x8 = bench.synth_batch(16, 0).to(DEV)
    pred = m.forward_augment(x8)[0]
    idx = [0, 15]
    got = pred[idx].float().cpu()
    x = x8[idx].cpu().float() / 255
    want, _ = tta_ref.forward_augment(m_cpu, x)
    emu, _ = tta_ref.forward_augment(m_cpu, x, emulate_bf16=True)
    branches, rows = tta_geometry(1024, 1024)
    assert got.shape == want.shape == (2, rows, 200)
    for g in branches:
        o = g["row_off"]
        for l in g["levels"]:
            r = g["level_rows"][l]
            gg, w, e = (t[:, o:o + r] for t in (got, want, emu))
            rel, floor = ((gg - w).norm() / w.norm()).item(), ((e - w).norm() / w.norm()).item()
            print(f"scale {g['scale']} level {l}: rel_l2 {rel:.3e}, bf16 floor {floor:.3e}")
            assert rel < 2.0 * floor + 3e-3, (g["scale"], l, rel, floor)
            o += r
        assert o == g["row_off"] + g["rows"]
    cw = want[..., 4] > bench.CONF

    def iou(t):
        c = t[..., 4] > bench.CONF
        return (c & cw).sum().item() / max((c | cw).sum().item(), 1)

    print("obj mask IoU", iou(got), "floor", iou(emu))
    assert iou(got) >= iou(emu) - 0.1


@pytest.mark.parametrize("size,B,S", [("n", 3, 160), ("s", 2, 256)])
def test_records_plus_nms_equal_tensor_plus_nms(size, B, S):
    m = build_mirror(size, nc=15, seed=3, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    x = torch.rand(B, 3, S, S + 32, generator=torch.Generator().manual_seed(2)).to(DEV)
    pred = m.forward_augment(x)[0].clone()
    rec = m.detect_records(x, augment=True)
    assert rec.data.shape == (B, pred.shape[1], 24) and rec.nc == 15
    pred, near_ties = check_records(pred, rec.data, 15)
    assert near_ties <= max(2, pred.shape[0] * pred.shape[1] // 1000)
    for kw in (dict(multi_label=True, max_det=300), dict(multi_label=False, max_det=100), dict(multi_label=True, classes=[1, 5])):
        a = general.non_max_suppression_obb(pred, 0.25, 0.45, **kw)
        b = general.non_max_suppression_obb(rec, 0.25, 0.45, **kw)
        assert sum(t.shape[0] for t in a) > 0
        for u, v in zip(a, b):
            assert torch.equal(u, v)


def _tta_composition(model, loader, kw, iouv, nc):
    from oracle import valmetrics_ref as V
    from yolov5_obb_b200.val import match_batch
    stats = []
    for im, targets, _, shapes in loader:
        dets, rows = general.non_max_suppression_obb(model.detect_records(im.to(DEV), augment=True), return_packed=True, **kw)
        t = targets.to(DEV)
        correct, _, _ = match_batch(dets, torch.tensor(rows, device=DEV), t, shapes, iouv.to(DEV), want_geometry=False)
        stats += V.image_stats(correct.cpu().numpy(), dets.cpu().numpy(), rows, targets.numpy(), iouv.numel())
    return V.val_metrics(V.concat_stats(stats), nc)


def test_validator_augment_equals_composition_of_public_calls():
    from tests.test_valmetrics_gpu import _loader, _model_and_batches, assert_same
    from yolov5_obb_b200.val import Validator
    model, batches = _model_and_batches()
    loader = _loader(model, batches, 0.1)
    v = Validator(model, conf_thres=0.1, iou_thres=0.4, max_det=300, augment=True)
    m = v(loader)
    want = _tta_composition(model, loader, v.nms, v.iouv.cpu(), model.model[-1].nc)
    assert m.seen == sum(b.shape[0] for b in batches) and v.reruns == 0
    assert_same(m, want)
    plain = Validator(model, conf_thres=0.1, iou_thres=0.4, max_det=300)(loader)
    assert not np.array_equal(np.array(m.results), np.array(plain.results))   # the augmented rows were really used


def test_validator_augment_reruns_overflowed_batches(monkeypatch):
    from tests.test_valmetrics_gpu import _loader, _model_and_batches, assert_same
    from yolov5_obb_b200.val import Validator
    model, batches = _model_and_batches(obj_bias=6.0)
    batches = batches[:2] + batches[:1]
    loader = _loader(model, batches, 0.01)
    monkeypatch.setattr(general, "_CAP_HINT", {})
    v = Validator(model, conf_thres=0.01, iou_thres=0.4, max_det=1500, augment=True)
    m = v(loader)
    assert v.reruns >= 1
    general._CAP_HINT.clear()
    want = _tta_composition(model, loader, v.nms, v.iouv.cpu(), model.model[-1].nc)
    assert m.seen == 5
    assert_same(m, want)


def test_pruned_plans_and_replan_after_update():
    m = build_mirror("s", nc=15, seed=2).to(DEV)
    x = torch.rand(2, 3, 256, 320, generator=torch.Generator().manual_seed(4)).to(DEV)
    plan = m.tta_plan(tuple(x.shape), DEV)
    l0, l1, l2 = (e.op_layers for e in plan.engines)
    assert not {21, 22, 23, ("Detect", 2)} & set(l0) and ("Detect", 0) in l0 and 20 in l0
    assert ("Detect", 0) not in l2 and {21, 23, ("Detect", 1), ("Detect", 2)} <= set(l2)
    assert {21, 23, ("Detect", 0), ("Detect", 1), ("Detect", 2)} <= set(l1)
    full = m.records_plan((2, 3, 256, 320), DEV)
    assert plan.engines[0].flops < full.flops and len(plan.engines[0].ops) < len(full.ops)
    before = m.forward_augment(x)[0].clone()
    with torch.no_grad():
        m.model[-1].m[1].bias.add_(0.25)
        m.model[4].cv1.bn.weight.mul_(1.1)
    after = m.forward_augment(x)[0].clone()
    assert not torch.equal(before, after)
    fresh = copy.deepcopy(m)
    assert torch.equal(after, fresh.forward_augment(x)[0])
    assert torch.equal(m.detect_records(x, augment=True).data, fresh.detect_records(x, augment=True).data)


def test_refusals(model_n):
    with pytest.raises(RuntimeError):
        model_n.forward_augment(torch.zeros(1, 3, 64, 64))               # CPU tensor
    with pytest.raises(RuntimeError):
        model_n.forward_augment(torch.zeros(1, 3, 72, 64, device=DEV))   # not a multiple of 32
    with pytest.raises(RuntimeError):
        model_n.detect_records(torch.zeros(1, 3, 64, 80, device=DEV), augment=True)
    model_n.train()
    try:
        with pytest.raises(RuntimeError):
            model_n.forward_augment(torch.zeros(1, 3, 64, 64, device=DEV))
        with pytest.raises(RuntimeError):
            model_n.detect_records(torch.zeros(1, 3, 64, 64, device=DEV), augment=True)
    finally:
        model_n.eval()
    with pytest.raises(RuntimeError):
        model_n(torch.zeros(1, 3, 64, 64, device=DEV), augment=True)    # Model.forward(augment=True) still refuses
