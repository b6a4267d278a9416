"""GPU test of the host-to-host detection pipeline (pipeline.DetectPipeline = the loop of detect.py:104-122 /
val.py:183-207): the two-deep software pipeline (async H2D / async D2H) must yield, batch by batch, exactly what the
blocking calls model(x) + non_max_suppression_obb(pred) give; and the packed / async return forms of
non_max_suppression_obb are the same rows as the list form."""
import pytest
import torch

from tests.modelgen import build_mirror
from tests.tilegen import synth_tiles

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("slots,fused", [(1, True), (2, True), (3, True), (2, False)])
def test_pipeline_equals_blocking_calls(slots, fused):
    """slots batches in flight on their own streams (own plan and post-process graph each): every batch - all distinct -
    must come back in order with exactly the blocking calls' rows; 7 batches so that every slot is used after its graphs
    were captured (third use) and the pinned result slots wrap around."""
    from yolov5_obb_b200.general import non_max_suppression_obb
    from yolov5_obb_b200.pipeline import DetectPipeline
    m = build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    batches = [synth_tiles(2, 256, seed=s).pin_memory() for s in range(1, 4 * slots + 2)]
    kw = dict(conf_thres=0.25, iou_thres=0.45, multi_label=True, max_det=300)
    want = []
    for xb in batches:
        pred, _ = m(xb.to(DEV))
        dets = non_max_suppression_obb(pred, **kw)
        packed, counts = non_max_suppression_obb(pred, return_packed=True, **kw)
        out, cdev, cap = non_max_suppression_obb(pred, return_packed="async", **kw)
        c = cdev.tolist()
        assert c[2] <= cap, (c, cap)
        assert c[:2] == counts == [d.shape[0] for d in dets], (c, counts, [d.shape[0] for d in dets])
        for b in range(2):
            assert torch.equal(packed[b, :counts[b]], dets[b]) and torch.equal(out[b, :counts[b]], dets[b])
        if fused:   # the pipeline's own entry point, blocking (the tensor path's rows equal it up to theta near-ties: below)
            dets = non_max_suppression_obb(m.detect_records(xb.to(DEV)), **kw)
        want.append([d.cpu() for d in dets])
    pipe = DetectPipeline(m, 0.25, 0.45, 300, multi_label=True, device=DEV, slots=slots, fused_detect=fused)
    assert pipe.slots == (slots if fused else 1)
    got = list(pipe(iter(batches)))
    assert len(got) == len(want)
    assert sum(d.shape[0] for w in want for d in w) > 0
    for g, w in zip(got, want):
        assert len(g) == len(w)
        for a, b in zip(g, w):
            assert not a.is_cuda and torch.equal(a, b)
    assert pipe.h2d_bytes == sum(x.numel() for x in batches)


class _NoHint(dict):
    """A general._CAP_HINT that never learns: every async NMS starts from the optimistic capacity again."""

    def __setitem__(self, key, value):
        pass


def test_overflowed_batches_are_rerun_in_both_forms(monkeypatch):
    """conf_thres=0 with multi_label: every (anchor, class) pair of a 2 x 256^2 batch is a candidate, 2 * 4032 * 15 = 120,960
    against the optimistic capacity of 65,536, so the async NMS of every batch overflows and the pipeline re-runs it blocking.
    Both forms, two slots on one pipeline: each yielded batch must still equal the blocking calls, in order."""
    from tests.letterboxgen import synth_image
    from yolov5_obb_b200 import general
    from yolov5_obb_b200 import letterbox as lb
    from yolov5_obb_b200 import pipeline as P
    monkeypatch.setattr(general, "_CAP_HINT", _NoHint())
    nms = general.non_max_suppression_obb
    reruns = []

    def counting_nms(pred, **kw):
        reruns.append(kw.get("return_packed") is True)
        return nms(pred, **kw)

    monkeypatch.setattr(P, "non_max_suppression_obb", counting_nms)
    m = build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    kw = dict(conf_thres=0.0, iou_thres=0.45, multi_label=True, max_det=300)
    pipe = P.DetectPipeline(m, device=DEV, slots=2, **kw)

    batches = [synth_tiles(2, 256, seed=s).pin_memory() for s in range(1, 5)]
    want = [[d.cpu() for d in nms(m.detect_records(xb.to(DEV)), **kw)] for xb in batches]
    got = list(pipe(iter(batches)))
    assert sum(reruns) == len(batches) == len(got)
    for g, w in zip(got, want):
        assert len(g) == len(w) and all(torch.equal(a, b) for a, b in zip(g, w))

    images = [synth_image(256, 256, 30 + k) for k in range(8)]
    order, shapes = lb.rect_batch_shapes([(256, 256)] * len(images), 2, 256, 32, 0.0)
    want = [None] * len(images)
    for b, (Hp, Wp) in enumerate(shapes.tolist()):
        idx = [int(k) for k in order[2 * b:2 * b + 2]]
        places = [lb.place_rect(256, 256, 256, (Hp, Wp)) for _ in idx]
        batch = lb.pack_batch([images[k] for k in idx], places, Hp, Wp)
        eng = m.records_plan((2, 3, Hp, Wp), DEV)
        lb.letterbox_s2d(batch.host[:batch.nbytes].to(DEV), batch, eng.x_s2d, 1)
        packed, counts = nms(general.DetectRecords(eng.forward_s2d(), eng.nc, eng.half), return_packed=True, **kw)
        pad_gain = torch.tensor([p.pad_gain for p in places], dtype=torch.float32, device=DEV)
        polys = lb.scale_polys_batched(packed, torch.tensor(counts, device=DEV), pad_gain).cpu()
        for i, k in enumerate(idx):
            want[k] = (polys[i, :counts[i]], packed[i, :counts[i]].cpu())
    reruns.clear()
    got = list(pipe.run_images(images, img_size=256, stride=32, auto=False, batch_size=2))
    assert sum(reruns) == len(shapes) and len(got) == len(images)
    assert sum(r.shape[0] for _, r in want) > 0
    for g, (poly, rows) in zip(got, want):
        assert torch.equal(g.rows, rows) and torch.equal(g.polys, poly)


def test_submit_fork_join_device_resident():
    """DetectPipeline.submit: device-resident batches round-robin over the slot streams, bracketed by fork() / join(); each
    slot's last result equals the blocking call on that batch (distinct batches, so a slot mix-up cannot pass)."""
    from yolov5_obb_b200.general import non_max_suppression_obb
    from yolov5_obb_b200.pipeline import DetectPipeline
    m = build_mirror("n", nc=15, seed=0, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to(DEV)
    xs = [synth_tiles(2, 256, seed=s).to(DEV) for s in range(1, 9)]
    kw = dict(conf_thres=0.25, iou_thres=0.45, multi_label=True, max_det=300)
    want = [non_max_suppression_obb(m.detect_records(x), **kw) for x in xs]
    want = [[d.clone() for d in w] for w in want]
    pipe = DetectPipeline(m, 0.25, 0.45, 300, multi_label=True, device=DEV, slots=2)
    pipe.fork()
    outs = []
    for i, x in enumerate(xs):
        o = pipe.submit(x)
        if i >= len(xs) - 2:
            outs.append((i, o))
    pipe.join()
    torch.cuda.synchronize()
    for i, (packed, counts, cap) in outs:
        c = counts.tolist()
        assert 0 <= c[2] <= cap
        for b in range(2):
            assert torch.equal(packed[b, :c[b]], want[i][b])
    assert sum(d.shape[0] for w in want for d in w) > 0


@pytest.mark.parametrize("size,B,S", [("n", 3, 160), ("s", 2, 256)])
def test_fused_detect_records_equal_forward_plus_nms(size, B, S):
    """Model.detect_records (Detect epilogue writes compact (box, obj, cls, theta index) records) + the post-process gives
    the detections of Model.forward + non_max_suppression_obb on the [B, A, no] tensor: the records hold exactly the tensor's
    box / obj / class values (same sigmoid / decode arithmetic) and the index of the first maximum of the 180 theta logits -
    the tensor's argmax except between logits closer than the tensor's tanh.approx error (tests/recordcheck.py bounds that
    and patches those rows, after which the two detection lists must be bit-identical)."""
    import torch
    from tests.modelgen import build_mirror
    from yolov5_obb_b200.general import non_max_suppression_obb
    m = build_mirror(size, nc=15, seed=3, obj_bias=1.0, cls_bias=-1.0, det_gain=6.0).to("cuda:0")
    x = torch.rand(B, 3, S, S + 32, generator=torch.Generator().manual_seed(2)).to("cuda:0")
    pred, _ = m(x)
    pred = pred.clone()
    rec = m.detect_records(x)
    assert rec.data.shape == (B, pred.shape[1], 24) and rec.nc == 15
    from tests.recordcheck import check_records
    pred, near_ties = check_records(pred, rec.data, 15)
    assert near_ties <= max(2, pred.shape[0] * pred.shape[1] // 1000)
    for kw in (dict(multi_label=True, max_det=300), dict(multi_label=False, max_det=100), dict(multi_label=True, classes=[1, 5])):
        a = non_max_suppression_obb(pred, 0.25, 0.45, **kw)
        b = non_max_suppression_obb(rec, 0.25, 0.45, **kw)
        assert sum(t.shape[0] for t in a) > 0
        for u, v in zip(a, b):
            assert torch.equal(u, v)
