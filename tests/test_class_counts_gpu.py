"""The Detect head, the training loss, the validation loss and NMS at the class counts of real OBB datasets, against the
references the nc = 15 tests use.

The class count sets the Detect row width no = nc + 185 (a multiple of 4 only for nc = 3 mod 4), the compact record width
rec_w = roundup4(nc + 6), the Detect N tile NI = roundup32(roundup16(no)) and so which records kernel runs:

    nc   no (% 4)  rec_w  records kernel   why
     1   186 (2)     8    <192, true>      HRSC2016; every nc == 1 branch (no lcls, no multi-label, no class split)
     2   187 (3)     8    <192, true>      UCAS-AOD
     3   188 (0)    12    <192, true>      NI = 192 with 16-byte rows
    15   200 (0)    24    <224, true>      DOTA v1.0, the benchmarked count
    16   201 (1)    24    <224, true>      DOTA v1.5
    18   203 (3)    24    <224, true>      DOTA v2.0
    37   222 (2)    44    <224, true>      FAIR1M; the widest NI = 224 tile
    43   228 (0)    52    <256, true>      NI = 256 with 16-byte rows
    58   243 (3)    64    <256, true>      a record fills the 64-column staging row exactly
    59   244 (0)    68    generic          the first count that falls back to the shared epilogue
    64   249 (1)    72    generic          NMS's upper limit

Raw and decoded Detect rows whose width is not a multiple of 4 are stored element by element; everything the kernels write
is checked against a sentinel-filled destination, so a store that runs into the next row or past the region fails."""
import copy
import math

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from oracle.postprocess import non_max_suppression_obb as oracle_nms
from tests import test_conv_plans_exact_gpu as CE
from tests import test_detect_records_gpu as DR
from tests import test_valloss_gpu as VL
from tests.losscases import FakeModel
from tests.lossgen import compact_layouts, synth_preds, synth_targets
from tests.modelgen import build_mirror
from tests.predgen import synth_pred
from tests.recordcheck import check_records
from tests.test_engine_gpu import _compare
from tests.test_loss_exact_gpu import _check, _report
from tests.test_train_backward_gpu import _teacher_forced
from tests.test_train_step_gpu import _oracle_trajectory
from tests.tilegen import synth_tiles
from yolov5_obb_b200 import general
from yolov5_obb_b200.conv import DETECT_GENERIC, MODE_DETECT
from yolov5_obb_b200.engine import InferenceEngine, TTAPlan
from yolov5_obb_b200.loss import ComputeLoss
from yolov5_obb_b200.train_backward import BackwardPlan
from yolov5_obb_b200.train_engine import TrainEngine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NCS = (1, 2, 3, 15, 16, 18, 37, 43, 58, 59, 64)
PAD_ROWS = 3   # sentinel rows before and after the Detect region (3 * no floats: only 4-byte aligned when no % 4 != 0)


def _rec_w(nc):
    return (nc + 6 + 3) // 4 * 4


# ---- 1. every Detect launch exact ------------------------------------------------------------------------------------
def _plan_ops(nc, kind, H, W, full):
    """(conv ops, wgrad ops) of the yolov5n B = 2 plan of `kind`: the Detect launches and their backward parts, or every
    launch (full)."""
    B = 2
    m = build_mirror("n", nc=nc, seed=0)
    if kind == "train":
        m = m.train().to(DEV)
        eng = TrainEngine(m, B, H, W, DEV)
        plan = BackwardPlan(eng)
        parts = plan.det_parts + (plan.conv_parts if full else [])
        convs = ([lay.conv for lay in eng.conv_layers] if full else []) + list(eng.det_convs)
        for part in parts:
            convs += part.get("dgrad_ops", [])
        assert all(cv.desc.det_no == nc + 185 and cv.desc.det_decode == 0 for cv in eng.det_convs)
        return convs, [part["wgrad"] for part in parts], (eng, plan)
    compact = kind != "forward"
    det = m.model[-1]
    rows = det.na * sum((H // s) * (W // s) for s in (8, 16, 32))
    width = _rec_w(nc) if compact else det.no
    out = torch.empty((B, PAD_ROWS + rows + PAD_ROWS, width), dtype=torch.float32, device=DEV)
    eng = InferenceEngine(m, B, H, W, DEV, conv_flags=DETECT_GENERIC if kind == "records-generic" else 0,
                          compact_detect=compact, det_out=out, det_row_base=PAD_ROWS)
    convs = [op for op in eng.convs if full or op.desc.mode == MODE_DETECT]
    assert sum(op.desc.mode == MODE_DETECT for op in convs) == 3
    return convs, [], (eng,)


def _check_plan(nc, kind, H, W, full=False):
    torch.manual_seed(nc)
    convs, wgrads, keep = _plan_ops(nc, kind, H, W, full)
    st = CE._stats()
    for i, op in enumerate(convs):
        CE.check_conv(op, st, f"nc {nc} {kind} {H}x{W} conv {i}")
    for i, wg in enumerate(wgrads):
        CE.check_wgrad(wg, st, f"nc {nc} {kind} {H}x{W} wgrad {i}")
    print(f"\nnc {nc} {kind} {H}x{W}: {st['conv']} conv and {st['wgrad']} wgrad launches, {st['bitwise']} bitwise, "
          f"{st['tolerance']} within the epilogue bound (worst {st['worst']:.3f})"
          + (f", theta ties in {st['ties']} of {st['rows']} record rows" if kind.startswith("records") else ""))
    assert st["conv"] == len(convs) and st["wgrad"] == len(wgrads)
    if kind.startswith("records"):
        assert st["ties"] > 0
    if kind == "train":
        assert len(wgrads) >= 3 and any(wg.desc.co_group == nc + 185 and wg.desc.co_group_pad == (nc + 185 + 15) // 16 * 16
                                        for wg in wgrads)


@pytest.mark.parametrize("H,W", [(96, 160), (320, 256)])
@pytest.mark.parametrize("kind", ["forward", "records", "records-generic", "train"])
@pytest.mark.parametrize("nc", NCS)
def test_detect_launches_exact(nc, kind, H, W):
    """The Detect launches (and, for train, the Detect dgrad and wgrad with the (no, bn) padded channel groups) of the yolov5n
    plans against their descriptors (tests/convref.py), with every element outside the write mask unchanged."""
    _check_plan(nc, kind, H, W)


@pytest.mark.parametrize("kind", ["forward", "records", "records-generic", "train"])
def test_full_plan_exact_nc16(kind):
    """Every launch of the yolov5n B = 2 96x160 plans at nc = 16 (no = 201)."""
    _check_plan(16, kind, 96, 160, full=True)


# ---- 2. records epilogue against the generic epilogue ----------------------------------------------------------------
@pytest.mark.parametrize("B,H,W", [(2, 1024, 1024), (2, 768, 1024)])
@pytest.mark.parametrize("nc", [1, 3, 16, 37, 43, 58])
def test_records_match_generic_epilogue(nc, B, H, W):
    th = DR._records("s", B, H, W, nc=nc)
    assert bool((th == th.round()).all()) and float(th.min()) >= 0 and float(th.max()) < 180
    assert th.unique().numel() > 20


# ---- 3. the training loss against fp64 ------------------------------------------------------------------------------
@pytest.mark.parametrize("tcols", [187, 8, 7])
@pytest.mark.parametrize("nc", [1, 2, 16, 37, 64])
def test_loss_exact(nc, tcols):
    """Items, loss and every dense gradient element against tests/lossref.py, for grad_loss 1 and 2^16.  At nc = 1 the
    reference skips the class BCE (`if self.nc > 1`): lcls and every class-logit gradient are exactly 0."""
    B, S = 3, 256
    p = synth_preds(B, S, no=nc + 185, seed=nc)
    tg = compact_layouts(torch.from_numpy(synth_targets(B, 60, S, nc=nc, seed=nc)))[tcols]
    hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, nc, S)
    cl = ComputeLoss(FakeModel(hyp, nc=nc))
    bnd, worst, sec = _check(cl, p, tg, hyp, nc)
    _report(f"nc {nc}, {tcols}-column targets", bnd, worst, sec)
    assert sum(bnd["nrows"]) > 0
    pd = [x.to(DEV).requires_grad_(True) for x in p]
    loss, items = cl(pd, tg.to(DEV))
    grads = torch.autograd.grad(loss, pd)
    assert (float(items[2]) == 0.0) == (nc == 1)
    if nc == 1:
        assert all(not bool(g[..., 5].any()) for g in grads)


# ---- 4. validation-loss head items -----------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [1, 2, 16])
def test_head_items_bit_equal_to_loss_on_materialised_logits(nc, monkeypatch):
    """k_head_rows / k_head_obj's logits from the Detect inputs against ComputeLoss on the materialised head output, with
    exact (integer) logits: loss and items bit for bit, for 187-, 8- and 7-column targets."""
    monkeypatch.setattr(VL, "NO", nc + 185)
    B, H, W = 2, 256, 320
    cl = ComputeLoss(FakeModel(loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, nc, W), nc=nc))
    levels, ps = VL._integer_head(B, H, W, VL.CHANNELS["n"], seed=nc)
    for c, t in compact_layouts(torch.from_numpy(synth_targets(B, 40, H, nc=nc, seed=nc))).items():
        rc, loss, items, _ = VL._forward_head(cl, levels, t.to(DEV), B)
        assert rc == 0
        want_loss, want_items = cl(ps, t.to(DEV))
        assert torch.equal(loss, want_loss.detach()) and torch.equal(items, want_items), (c, items, want_items)
        assert (float(items[2]) == 0.0) == (nc == 1)


# ---- 5. post-process --------------------------------------------------------------------------------------------------
def _records_of(pred, nc):
    """The compact records (cx, cy, w, h, obj, cls[nc], first-maximum theta index, zero padding) of [B, A, nc + 185] rows."""
    rec = torch.zeros(pred.shape[:2] + (_rec_w(nc),), dtype=torch.float32, device=pred.device)
    rec[..., :5 + nc] = pred[..., :5 + nc]
    rec[..., 5 + nc] = pred[..., 5 + nc:].argmax(-1).float()
    return general.DetectRecords(rec, nc)


@pytest.mark.parametrize("nc", [1, 2, 16, 64])
def test_nms_matches_oracle(nc, ref_ext):
    """non_max_suppression_obb on the device against oracle/postprocess.py with multi_label on and off, agnostic on and off,
    and the class split on and off; records built from the same rows give the same output as the tensor.

    Rows against the per-image loop over the reference's own CUDA kernel, with test_postprocess_gpu's allowance (a decisive IoU
    within FMA distance of the threshold may flip one box); against the CPU oracle, whose IoU rounds differently, the kept
    counts differ by at most one and all but two rows are equal."""
    from oracle.postprocess import ref_obb_nms_cuda
    B, A = 2, 6000
    pred = synth_pred(B, A, nc, seed=40 + nc, frac_obj=0.05)
    pd = torch.from_numpy(pred).to(DEV)
    rec = _records_of(pd, nc)
    n = 0
    for multi in (True, False):
        for agnostic in (False, True):
            kw = dict(conf_thres=0.25, iou_thres=0.45, multi_label=multi, agnostic=agnostic, max_det=1500)
            exp = oracle_nms(pd, nms_mode=1, nms_fn=ref_obb_nms_cuda(ref_ext), **kw)
            cpu = oracle_nms(torch.from_numpy(pred), nms_mode=1, **kw)
            for nosplit in (False, True):
                general._NO_SPLIT.clear()
                if nosplit:
                    general._NO_SPLIT[(B, A, nc)] = True
                try:
                    got = general.non_max_suppression_obb(pd, **kw)
                    got_rec = general.non_max_suppression_obb(rec, **kw)
                finally:
                    general._NO_SPLIT.clear()
                for b in range(B):
                    what = (kw, nosplit, b)
                    g, e, c = got[b].cpu().numpy(), exp[b].cpu().numpy(), cpu[b].numpy()
                    assert g.shape == e.shape, (what, g.shape, e.shape)
                    # the eager loop forms theta with ATen's own rounding: one fp32 ulp apart; every other column exact
                    same = ((np.delete(g, 4, 1) == np.delete(e, 4, 1)).all(1)
                            & np.isclose(g[:, 4], e[:, 4], rtol=2 ** -22, atol=0))
                    assert same.mean() > 0.995, (what, same.mean())
                    common = len({r.tobytes() for r in g} & {r.tobytes() for r in c})
                    assert abs(len(g) - len(c)) <= 1 and common >= max(len(g), len(c)) - 2, (what, len(g), len(c), common)
                    assert torch.equal(got[b], got_rec[b]), what
                    if nc == 1:
                        assert not bool(got[b][:, 6].any())
                    n += g.shape[0]
    assert n > 0


# ---- 6. end to end ----------------------------------------------------------------------------------------------------
def _theta_prior_removed(m):
    """The reference's bias prior log(0.6 / (nc - 0.99)) (_initialize_biases) also lands on the 180 theta bins: at nc = 1 it is
    +13.3, every theta sigmoid is 1.0 in fp32 and the theta arg-max of every row is a tie.  Taking it off the theta bins (the
    same model on both sides of the comparison) leaves a theta arg-max to compare."""
    det = m.model[-1]
    with torch.no_grad():
        for mi in det.m:
            mi.bias.view(det.na, det.no)[:, 5 + det.nc:] -= math.log(0.6 / (det.nc - 0.999999))
    return m


@pytest.mark.parametrize("nc", [16, 1])
def test_eval_forward_matches_fp32_oracle(nc):
    m = _theta_prior_removed(build_mirror("n", nc=nc, seed=1))
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(5))
    ref, _ = model_ref.forward(m, x)
    pred, _ = m.to(DEV)(x.to(DEV))
    torch.cuda.synchronize()
    assert pred.shape == ref.shape and pred.shape[-1] == nc + 185
    _compare(pred, ref, f"yolov5n nc {nc} vs fp32 oracle", nc=nc)


@pytest.mark.parametrize("nc", [16, 1])
def test_records_plus_nms_equal_tensor_plus_nms(nc):
    # one class has no second chance to pass conf_thres: a positive class bias gives nc = 1 candidates too
    m = _theta_prior_removed(build_mirror("n", nc=nc, seed=3, obj_bias=1.0, cls_bias=-1.0 if nc > 1 else 1.0,
                                          det_gain=6.0)).to(DEV)
    x = torch.rand(2, 3, 256, 320, generator=torch.Generator().manual_seed(2)).to(DEV)
    pred = m(x)[0].clone()
    rec = m.detect_records(x)
    assert rec.data.shape[-1] == _rec_w(nc)
    pred, near_ties = check_records(pred, rec.data, nc)
    assert near_ties <= max(2, pred.shape[0] * pred.shape[1] // 1000)
    for kw in (dict(multi_label=True, max_det=300), dict(multi_label=False, max_det=100)):
        a = general.non_max_suppression_obb(pred, 0.25, 0.45, **kw)
        b = general.non_max_suppression_obb(rec, 0.25, 0.45, **kw)
        assert sum(t.shape[0] for t in a) > 0
        for u, v in zip(a, b):
            assert torch.equal(u, v)


@pytest.mark.parametrize("nc", [16, 1])
def test_train_forward_matches_oracle(nc):
    """test_train_forward_gpu's rule: per Detect level the relative L2 distance to the fp32 oracle below 1.5x that of the
    bf16-emulating oracle + 3e-3."""
    m = build_mirror("n", nc=nc, seed=2).train()
    x = torch.rand(2, 3, 128, 160, generator=torch.Generator().manual_seed(8))
    emu = model_ref.forward(copy.deepcopy(m), x, training=True, emulate_bf16=True)
    want = model_ref.forward(copy.deepcopy(m), x, training=True)
    with torch.no_grad():
        got = m.to(DEV)(x.to(DEV))
    for l, (a, b, f) in enumerate(zip(got, want, emu)):
        assert a.shape == b.shape and a.shape[-1] == nc + 185
        rel = ((a.cpu() - b).norm() / b.norm()).item()
        floor = ((f - b).norm() / b.norm()).item()
        print(f"nc {nc} level {l}: rel L2 {rel:.4g}, bf16-storage noise floor {floor:.4g}")
        assert rel < 1.5 * floor + 3e-3


@pytest.mark.parametrize("nc", [16, 1])
def test_backward_teacher_forced_parity(nc):
    """test_train_backward_gpu's one-module-deep teacher forcing and tolerances."""
    m = build_mirror("n", nc=nc, seed=3).train()
    ref_m = copy.deepcopy(m)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(2, 3, 128, 160, generator=g)
    md = m.to(DEV)
    outs = md(x.to(DEV))
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
    print(f"nc {nc}: {len(rels)} parameter tensors: median rel {rels[len(rels) // 2]:.3g}, max {rels[-1]:.3g}")
    assert not bad, bad[:10]
    assert rels[len(rels) // 2] < 2e-2
    grels = [((gout(i) - ref).norm().item() / max(ref.norm().item(), 1e-12), i) for i, ref in sorted(gl.items())]
    assert max(r for r, _ in grels) < 6e-2, grels
    for i, (want, have) in inner.items():
        assert (have - want).norm().item() / max(want.norm().item(), 1e-12) < 3e-2


@pytest.mark.parametrize("nc", [16, 1])
def test_loss_trajectory_against_the_cpu_oracle(nc):
    """Three SGD steps of yolov5n at 128^2 on one batch, with test_train_step_gpu's yardstick: step 0 to 1e-3, then within 3x
    the bf16-emulating oracle's own drift + 2 % of the loss."""
    from yolov5_obb_b200.train_step import TrainStep
    B, S, N = 4, 128, 3
    m0 = build_mirror("n", nc=nc, seed=1).train()
    imgs = synth_tiles(B, S, seed=3)
    tg = torch.from_numpy(synth_targets(B, 40, S, nc=nc, seed=3))
    ref = _oracle_trajectory(m0, imgs, tg, N, S, emulate_bf16=False)
    emu = _oracle_trajectory(m0, imgs, tg, N, S, emulate_bf16=True)
    ts = TrainStep(copy.deepcopy(m0).to(DEV), batch_size=64, imgsz=S)
    dev = [ts.step(imgs.to(DEV), tg.to(DEV))[0].item() for _ in range(N)]
    print(f"nc {nc}: oracle fp32 {ref}, oracle bf16 {emu}, device {dev}")
    assert abs(dev[0] - ref[0]) < 1e-3 * abs(ref[0]) + 2e-2 * abs(emu[0] - ref[0]) + 1e-3
    run_max = 0.0
    for i in range(N):
        run_max = max(run_max, abs(emu[i] - ref[i]))
        assert abs(dev[i] - ref[i]) < 3.0 * run_max + 0.02 * abs(ref[i]) + 1e-3, (i, dev[i], ref[i], emu[i])


# ---- 7. refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc", [65, 72])
def test_refuses_class_counts_past_64(nc):
    """nc = 72 would also give det_no = 257, past the 256-column N tile."""
    m = build_mirror("n", nc=nc, seed=0)
    assert m.model[-1].no == nc + 185
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        InferenceEngine(m, 1, 64, 64, DEV)
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        TTAPlan(m, 1, 64, 64, DEV)
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        TrainEngine(m.train(), 1, 64, 64, DEV)
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        ComputeLoss(FakeModel(loss_ref.DEFAULT_HYP, nc=nc))
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        general.non_max_suppression_obb(torch.rand(1, 10, nc + 185, device=DEV))


def test_refuses_zero_classes():
    """Model falls back to the yaml's count for a falsy nc, so nc = 0 is only reachable through a Detect or a tensor."""
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        ComputeLoss(FakeModel(loss_ref.DEFAULT_HYP, nc=0))
    with pytest.raises(RuntimeError, match=r"1\.\.64"):
        general.non_max_suppression_obb(torch.rand(2, 10, 185, device=DEV))
