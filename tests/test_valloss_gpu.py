"""GPU tests of the validation loss from the Detect inputs (y5obb_loss_forward_head, ComputeLoss.head_items, Validator with
compute_loss): bit-exact against ComputeLoss on the materialised head output when every logit is exact, the seeded records plan
against the fp32 oracle, the REFERENCE golden (tests/golden/valloss_golden.npz), the Validator's 8-tuple, and the refusals."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from tests import vallossgen as VG
from tests.losscases import FakeModel
from tests.lossgen import boundary_targets, synth_targets
from yolov5_obb_b200 import _lib, general
from yolov5_obb_b200.loss import ComputeLoss, LossHead, compact_csl_index
from yolov5_obb_b200.val import Validator

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STRIDES = (8, 16, 32)
NA, NO = 3, 200
CHANNELS = {"n": (64, 128, 256), "s": (128, 256, 512), "m": (192, 384, 768), "x": (320, 640, 1280)}


def _hyp(imgsz):
    return loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, 15, imgsz)


def _integer_head(B, H, W, Cs, seed):
    """Integer-valued bf16 features (pixel stride C + 8, so not dense), weights and fp32 biases with sum |f * w| < 2^24: every
    logit is exact in any summation order.  Returns (per level (feature view, weight, bias), materialised [B, na, h, w, no])."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    levels, ps = [], []
    for s, C in zip(STRIDES, Cs):
        h, w = H // s, W // s
        buf = torch.randint(-2, 3, (B, h, w, C + 8), generator=g, device=DEV)
        buf *= torch.rand(buf.shape, generator=g, device=DEV) < 0.25
        f = buf.to(torch.bfloat16)[..., :C]
        wt = torch.randint(-1, 2, (NA * NO, C), generator=g, device=DEV)
        wt *= torch.rand(wt.shape, generator=g, device=DEV) < 0.125
        wt = wt.to(torch.bfloat16)
        bias = torch.randint(-4, 5, (NA * NO,), generator=g, device=DEV).float()
        assert 2 * C + 4 < 2 ** 24   # |f| <= 2, |w| <= 1, |bias| <= 4
        logit = (f.double().reshape(-1, C) @ wt.double().T + bias.double()).float()
        ps.append(logit.view(B, h, w, NA, NO).permute(0, 3, 1, 2, 4).contiguous())
        levels.append((f, wt, bias))
    return levels, ps


def _forward_head(cl, levels, tg, B):
    d = cl._base_desc(B, NO, tg)
    h = LossHead()
    for i, (f, w, b) in enumerate(levels):
        h.feat[i] = f.data_ptr()
        h.pix_stride[i], h.row_stride[i], h.img_stride[i] = f.stride(2), f.stride(1), f.stride(0)
        h.H[i], h.W[i], h.C[i] = f.shape[1], f.shape[2], f.shape[3]
        h.w[i], h.bias[i] = w.data_ptr(), b.data_ptr()
    L = _lib.lib()
    nbytes = L.y5obb_loss_head_workspace_bytes(ctypes.byref(d), ctypes.byref(h))   # 0 = refused
    ws = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=DEV)
    loss = torch.empty(1, device=DEV)
    items = torch.empty(4, device=DEV)
    rc = L.y5obb_loss_forward_head(ctypes.byref(d), ctypes.byref(h), loss.data_ptr(), items.data_ptr(), ws.data_ptr(),
                                   ws.numel(), _lib.stream_ptr(DEV))
    return rc, loss, items, (d, h, nbytes)


def _layouts(tg):
    """The 187-, 8- and 7-column forms of the same targets."""
    t8 = torch.cat([tg[:, :7], torch.from_numpy(compact_csl_index(tg[:, 6].double().numpy())).view(-1, 1)], 1)
    return {187: tg, 8: t8, 7: tg[:, :7].contiguous()}


def _assert_exact(B, H, W, Cs, tg, seed, cols=(187,)):
    cl = ComputeLoss(FakeModel(_hyp(max(H, W))))
    levels, ps = _integer_head(B, H, W, Cs, seed)
    for c in cols:
        t = _layouts(tg)[c].to(DEV)
        rc, loss, items, _ = _forward_head(cl, levels, t, B)
        assert rc == 0
        want_loss, want_items = cl(ps, t)
        assert torch.equal(loss, want_loss.detach()) and torch.equal(items, want_items), (c, items, want_items)
        assert torch.isfinite(items).all()
    return items


@pytest.mark.parametrize("size", sorted(CHANNELS))
def test_exact_b16_1024(size):
    B = 16
    tg = torch.from_numpy(synth_targets(B, B * 23, 1024, seed=11))
    items = _assert_exact(B, 1024, 1024, CHANNELS[size], tg, seed=5)
    assert (items > 0).all()


def test_exact_320x256_layouts_and_duplicates():
    """P5 of a 256 x 320 input has 80 cells per (image, anchor): the 256-cell obj blocks straddle anchors.  Rows repeated
    verbatim land in the same cells (the last writer wins tobj); every target layout.  Then targets on build_targets'
    boundaries (tests/lossgen.boundary_targets)."""
    B = 2
    tg = torch.from_numpy(synth_targets(B, 40, 256, seed=12))
    tg = torch.cat([tg, tg[5:9], tg[5:6]])
    _assert_exact(B, 256, 320, CHANNELS["s"], tg, seed=6, cols=(187, 8, 7))
    _assert_exact(B, 256, 320, CHANNELS["s"], torch.from_numpy(boundary_targets(B, 256, 320, seed=13)), seed=6,
                  cols=(187, 8, 7))


def test_exact_empty_targets():
    items = _assert_exact(3, 256, 320, CHANNELS["n"], torch.zeros((0, 187)), seed=7)
    assert items[1] > 0 and items[0] == 0 and items[2] == 0 and items[3] == 0


def _plan_model(size="s"):
    from tests.modelgen import build_mirror
    m = build_mirror(size, nc=15, seed=0, obj_bias=VG.OBJ_BIAS).to(DEV)
    m.hyp = _hyp(VG.HYP_IMGSZ)
    return m


def test_plan_head_items_match_oracle_on_plan_features():
    m = _plan_model("s")
    cl = ComputeLoss(m)
    im, tg = VG.batch(0)
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
    raw = model_ref.detect_fwd(det, feats, training=True)
    want_loss, want_items = loss_ref.compute_loss(raw, tg, det.anchors, det.stride, m.hyp, 15)
    np.testing.assert_allclose(items.cpu().numpy(), want_items.numpy(), rtol=1e-5, atol=0)
    np.testing.assert_allclose(loss.cpu().numpy(), want_loss.detach().numpy(), rtol=1e-5, atol=0)


@pytest.mark.parametrize("size", VG.SIZES)
def test_device_items_near_reference_golden(size):
    from pathlib import Path
    from tests.modelgen import build_mirror
    from tests.test_valloss_cpu import oracle_items
    G = np.load(Path(__file__).resolve().parent / "golden" / "valloss_golden.npz")
    gold = G[f"{size}/items"]
    emu = oracle_items(build_mirror(size, nc=15, seed=0, obj_bias=VG.OBJ_BIAS), emulate_bf16=True)
    m = _plan_model(size)
    cl = ComputeLoss(m)
    got = []
    for i in range(VG.N_BATCHES):
        im, tg = VG.batch(i)
        m.detect_records(im.to(DEV))
        got.append(cl.head_items(m.records_plan(tuple(im.shape), DEV), tg.to(DEV))[1].cpu().numpy())
    got = np.stack(got)
    bound = 2 * np.abs(emu - gold) + 1e-4 * np.abs(gold)
    assert np.all(np.abs(got - gold) <= bound), (got, gold, emu)


def _validator_setup(obj_bias=None):
    from tests.test_valmetrics_gpu import _loader, _model_and_batches
    model, batches = _model_and_batches(obj_bias)
    model.hyp = _hyp(512)
    return model, batches, _loader


def _per_batch_loss(model, cl, loader):
    acc = torch.zeros(4, device=DEV)
    for im, t, _, _ in loader:
        x = im.to(DEV)
        model.detect_records(x)
        acc += cl.head_items(model.records_plan(tuple(x.shape), DEV), t.to(DEV))[1]
    return tuple((acc.cpu() / len(loader)).tolist())


def _assert_validator(model, loader, **kw):
    cl = ComputeLoss(model)
    plain = Validator(model, **kw)(loader)
    v = Validator(model, compute_loss=cl, **kw)
    m = v(loader)
    assert len(m.results) == 8 and m.results[:4] == plain.results
    assert np.array_equal(m.maps, plain.maps) and np.array_equal(m.fitness(), plain.fitness())
    assert m.results[4:] == _per_batch_loss(model, cl, loader)
    assert all(r > 0 for r in m.results[4:5] + m.results[5:6])
    return v


def test_validator_results_with_loss():
    model, batches, _loader = _validator_setup()
    v = _assert_validator(model, _loader(model, batches, 0.1), conf_thres=0.1, iou_thres=0.4, max_det=300)
    assert v.reruns == 0


def test_validator_loss_with_overflow_reruns(monkeypatch):
    model, batches, _loader = _validator_setup(obj_bias=6.0)
    loader = _loader(model, batches[:2] + batches[:1], 0.01)
    monkeypatch.setattr(general, "_CAP_HINT", {})
    cl = ComputeLoss(model)
    v = Validator(model, conf_thres=0.01, iou_thres=0.4, max_det=1500, compute_loss=cl)
    m = v(loader)
    assert v.reruns == 2   # the re-run batches add their loss once
    general._CAP_HINT.clear()
    assert m.results[4:] == _per_batch_loss(model, cl, loader)


def test_refusals():
    from yolov5_obb_b200.engine import InferenceEngine
    from tests.modelgen import build_mirror
    m = _plan_model("n")
    cl = ComputeLoss(m)
    im, tg = VG.batch(0)
    x, t = im.to(DEV), tg.to(DEV)
    m.detect_records(x)
    plan = m.records_plan(tuple(x.shape), DEV)
    cl.head_items(plan, t)
    with pytest.raises(RuntimeError):
        Validator(m, augment=True, compute_loss=cl)
    with pytest.raises(RuntimeError):
        cl.head_items(plan, torch.zeros((3, 10), device=DEV))
    with pytest.raises(RuntimeError):
        cl.head_items(plan, tg)
    with pytest.raises(RuntimeError):
        cl.head_items(m.tta_plan(tuple(x.shape), DEV, compact_detect=True), t)
    with pytest.raises(RuntimeError):
        cl.head_items(InferenceEngine(m, 2, 256, 320, DEV, compact_detect=True, levels=(0, 1)), t)
    other = build_mirror("n", nc=10, seed=0)
    other.hyp = m.hyp
    with pytest.raises(RuntimeError):
        ComputeLoss(other).head_items(plan, t)
    shifted = FakeModel(m.hyp)
    shifted.model[0].anchors *= 1.5
    with pytest.raises(RuntimeError):
        ComputeLoss(shifted).head_items(plan, t)
    # the C ABI: C % 8, a null pointer
    levels, _ = _integer_head(1, 64, 64, (16, 16, 16), seed=1)
    cl15 = ComputeLoss(FakeModel(m.hyp))
    tg1 = torch.from_numpy(synth_targets(1, 4, 64, seed=1)).to(DEV)
    assert _forward_head(cl15, levels, tg1, 1)[0] == 0
    bad = [(levels[0][0][..., :12], levels[0][1][:, :12].contiguous(), levels[0][2])] + levels[1:]
    rc, _, _, (_, _, nbytes) = _forward_head(cl15, bad, tg1, 1)
    assert rc == 1 and nbytes == 0
    d, h, _ = _forward_head(cl15, levels, tg1, 1)[3]
    h.bias[2] = None
    assert _lib.lib().y5obb_loss_head_workspace_bytes(ctypes.byref(d), ctypes.byref(h)) == 0
