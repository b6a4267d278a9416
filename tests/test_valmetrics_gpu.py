"""GPU tests of the validation metrics (yolov5_obb_b200/val.py ValStats / Validator, csrc/val_metrics.cu): the reference's own
ap_per_class / fitness / val.py tail (tests/golden/valmetrics_golden.npz) bit for bit, the CPU restatement
oracle/valmetrics_ref.py on a tie-heavy set of 2M rows, the accumulation fed by match_batch, the Validator loop against the
composition of the blocking public calls, the NMS-overflow re-run, and the refusals."""
import numpy as np
import pytest
import torch

from oracle import valmetrics_ref as V
from tests.test_valmetrics_cpu import CASES, G, case_stats
from tests.valmetricsgen import synth_stats, val_batches
from yolov5_obb_b200 import general
from yolov5_obb_b200.val import ValStats, Validator, match_batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def as_batch(tp, conf, cls, tcls, image, row, images=None):
    """Rows with (image, row) positions -> one add() batch: dets [B, max_det, 7], counts, correct, targets (labels spread
    over the images).  `images` selects a subset of the images (their rows and labels)."""
    B = int(image.max()) + 1 if len(image) else 1
    max_det = int(row.max()) + 1 if len(row) else 1
    dets = np.zeros((B, max_det, 7), np.float32)
    correct = np.zeros((B, max_det, tp.shape[1]), bool)
    dets[image, row, 5], dets[image, row, 6] = conf, cls
    correct[image, row] = tp
    counts = np.bincount(image, minlength=B).astype(np.int64)
    timg = np.arange(len(tcls)) % B
    targets = np.stack([timg, tcls], 1).astype(np.float32)
    if images is not None:
        keep = np.isin(np.arange(B), images)
        counts[~keep] = 0
        targets = targets[np.isin(timg, images)]
    return [torch.from_numpy(a).to(DEV) for a in (dets, counts, correct, targets)]


def device_metrics(stats, image, row, nc, split=None):
    tp, conf, cls, tcls = stats
    vs = ValStats(nc, tp.shape[1], DEV)
    if split is None:
        vs.add(*as_batch(tp, conf, cls, tcls, image, row))
    else:   # the later images first, then the earlier ones at their own positions: appended out of order
        B = int(image.max()) + 1
        vs.seen = B
        vs.add(*as_batch(tp, conf, cls, tcls, image, row, np.arange(split, B)), image_base=0)
        vs.add(*as_batch(tp, conf, cls, tcls, image, row, np.arange(split)), image_base=0)
    return vs.metrics()


def assert_same(m, want):
    """ValMetrics against oracle.valmetrics_ref.val_metrics, every array equal."""
    assert np.array_equal(np.array(m.results), np.array(want["results"]))
    assert np.array_equal(m.maps, want["maps"]) and np.array_equal(m.ap_class, want["ap_class"])
    assert np.array_equal(m.p, want["p"]) and np.array_equal(m.r, want["r"])
    assert np.array_equal(m.ap50, want["ap50"]) and np.array_equal(m.ap, want["ap"])
    if "curves" in want:
        c = want["curves"]
        assert np.array_equal(m.p_curve, c["p_curve"]) and np.array_equal(m.r_curve, c["r_curve"])
        assert np.array_equal(m.ap_full, c["ap"])
        assert np.array_equal(m.tp, c["tp"]) and np.array_equal(m.fp, c["fp"]) and np.array_equal(m.f1, c["f1"])


@pytest.mark.parametrize("name,nc", [c for c in CASES if c[0] != "valgen"])
def test_device_equals_reference_golden(name, nc):
    m = device_metrics(case_stats(name), G[f"{name}/in/image"], G[f"{name}/in/row"], nc)
    assert np.array_equal(np.array(m.results), G[f"{name}/results"])
    assert np.array_equal(m.maps, G[f"{name}/maps"]) and np.array_equal(m.fitness(), G[f"{name}/fitness"])
    if f"{name}/ap_full" in G:
        for k in ("p_curve", "r_curve", "ap_full", "ap_class", "tp", "fp", "p", "r", "f1", "ap50", "ap"):
            assert np.array_equal(getattr(m, k), G[f"{name}/{k}"]), k
    else:
        assert m.ap_class.size == 0
    assert m.nt.sum() == len(G[f"{name}/in/target_cls"])


@pytest.fixture(scope="module")
def tie_set():
    classes = [(400_000, 1_100_000, None)] + [(int(n), int(n) * 6, None) for n in np.linspace(2000, 30000, 13)] + [(50, 0, None)]
    out = synth_stats(classes, niou=10, seed=5, n_images=1000, conf_levels=250)
    assert len(out[1]) >= 2_000_000 and (out[2] == 0).sum() > 1_000_000
    return out


@pytest.mark.parametrize("split", [None, 400])
def test_device_equals_restatement_on_tie_heavy_set(tie_set, split):
    tp, conf, cls, tcls, image, row = tie_set
    want = V.val_metrics([tp, conf, cls, tcls], 15)
    m = device_metrics([tp, conf, cls, tcls], image, row, 15, split)
    assert_same(m, want)
    assert 0.0 < m.results[3] < 1.0


def test_stats_fed_by_match_batch_equal_val_loop():
    """ValStats.add on match_batch's output reproduces the per-image stats val.py:209-250 builds (golden), in order."""
    iouv = torch.linspace(0.5, 0.95, 10, device=DEV)
    vs = ValStats(15, 10, DEV)
    for dets, counts, targets, shapes in val_batches():
        d, c, t = (torch.from_numpy(a).to(DEV) for a in (dets, counts, targets))
        correct, _, _ = match_batch(d, c, t, shapes, iouv, want_geometry=False)
        vs.add(d, c, correct, t)
    tp, conf, cls, key = (x.cpu().numpy() for x in vs.rows())
    assert np.array_equal(tp.astype(bool), G["valgen/stats/tp"]) and np.array_equal(conf, G["valgen/stats/conf"])
    assert np.array_equal(cls.astype(np.float32), G["valgen/stats/pred_cls"])
    assert np.array_equal(np.diff(key) > 0, np.ones(len(key) - 1, bool))
    want_nt = np.bincount(G["valgen/stats/target_cls"].astype(np.int64), minlength=15)
    assert np.array_equal(vs.nt.cpu().numpy(), want_nt) and vs.seen == 6
    m = vs.metrics()
    assert np.array_equal(np.array(m.results), G["valgen/results"]) and np.array_equal(m.maps, G["valgen/maps"])
    assert np.array_equal(m.p_curve, G["valgen/p_curve"]) and np.array_equal(m.ap_full, G["valgen/ap_full"])


def _model_and_batches(obj_bias=None):
    from tests.modelgen import build_mirror, calibrated_bench_model
    from tests.tilegen import synth_tiles
    m = (calibrated_bench_model("n", conf=0.1) if obj_bias is None else build_mirror("n", obj_bias=obj_bias)).to(DEV)
    shapes = [(2, 512, 512), (1, 512, 640), (2, 512, 512), (3, 384, 512)]
    batches = []
    for i, (B, H, W) in enumerate(shapes):
        im = synth_tiles(B, max(H, W), seed=40 + i)[:, :, :H, :W].contiguous()
        batches.append(im)
    return m, batches


def _targets_from(model, im, conf, seed):
    """Labels near the model's own confident detections (so that matches exist), some moved away, as val.py holds them."""
    recs = model.detect_records(im.to(DEV))
    dets, rows = general.non_max_suppression_obb(recs, conf, 0.4, multi_label=True, max_det=300, return_packed=True)
    rng = np.random.default_rng(seed)
    t = []
    for b, n in enumerate(rows):
        d = dets[b, :min(n, 40)].cpu().numpy()
        for r in d:
            jit = rng.normal(0, 2.0, 4) * (rng.random() < 0.7)
            t.append([b, r[6], r[0] + jit[0], r[1] + jit[1], r[2] + jit[2], r[3] + jit[3], r[4]])
    return torch.tensor(t, dtype=torch.float32).reshape(-1, 7)


def _composition(model, loader, kw, iouv, nc):
    """The blocking public calls chained as val.py:180-250 does, then the restatement."""
    stats = []
    for im, targets, _, shapes in loader:
        dets, rows = general.non_max_suppression_obb(model.detect_records(im.to(DEV)), return_packed=True, **kw)
        t = targets.to(DEV)
        counts = torch.tensor(rows, device=DEV)
        correct, _, _ = match_batch(dets, counts, t, shapes, iouv.to(DEV), want_geometry=False)
        stats += V.image_stats(correct.cpu().numpy(), dets.cpu().numpy(), rows, targets.numpy(), iouv.numel())
    return V.val_metrics(V.concat_stats(stats), nc)


def _loader(model, batches, conf):
    out = []
    for i, im in enumerate(batches):
        B, _, H, W = im.shape
        shapes = [((H, W), ((1.0, 1.0), (0.0, 0.0)))] * B
        out.append((im, _targets_from(model, im, max(conf, 0.1), i), [f"img{i}_{b}" for b in range(B)], shapes))
    return out


def test_validator_equals_composition_of_public_calls():
    model, batches = _model_and_batches()
    loader = _loader(model, batches, 0.1)
    v = Validator(model, conf_thres=0.1, iou_thres=0.4, max_det=300)
    m = v(loader)
    want = _composition(model, loader, v.nms, v.iouv.cpu(), model.model[-1].nc)
    assert m.seen == sum(b.shape[0] for b in batches) and v.reruns == 0
    assert_same(m, want)
    assert m.results[2] > 0.1
    m2 = v(loader)   # a second epoch on the same plans (the NMS post-process is graph-replayed by now)
    assert_same(m2, want)


def test_validator_reruns_overflowed_batches(monkeypatch):
    """With every anchor above conf_thres the async NMS overflows its first capacity: the batch is appended only by the
    blocking re-run, exactly once, and the result equals the composition of the blocking calls."""
    model, batches = _model_and_batches(obj_bias=6.0)
    batches = batches[:2] + batches[:1]
    loader = _loader(model, batches, 0.01)
    monkeypatch.setattr(general, "_CAP_HINT", {})   # (building the labels ran the blocking NMS, which raised it)
    v = Validator(model, conf_thres=0.01, iou_thres=0.4, max_det=1500)
    m = v(loader)
    assert v.reruns == 2   # the first two batches; the third has the first one's shape and the raised capacity
    general._CAP_HINT.clear()
    want = _composition(model, loader, v.nms, v.iouv.cpu(), model.model[-1].nc)
    assert m.seen == 5
    assert_same(m, want)


def test_refusals():
    tp, conf, cls, tcls, image, row = synth_stats(niou=10, seed=0)
    d, c, cor, t = as_batch(tp, conf, cls, tcls, image, row)
    vs = ValStats(8, 10, DEV)
    with pytest.raises(RuntimeError):
        vs.add(d.cpu(), c, cor, t)
    with pytest.raises(RuntimeError):
        vs.add(d.double(), c, cor, t)
    with pytest.raises(RuntimeError):
        vs.add(d, c.int(), cor, t)
    with pytest.raises(RuntimeError):
        vs.add(d, c, cor[..., :5], t)
    with pytest.raises(RuntimeError):
        vs.add(d, c, cor.float(), t)
    with pytest.raises(RuntimeError):
        vs.add(d, c, cor, t[:, :1].contiguous())
    with pytest.raises(RuntimeError):
        vs.add(d, c[:2], cor, t)
    with pytest.raises(RuntimeError):
        ValStats(8, 10, "cpu")
    ok = ValStats(8, 10, DEV)
    ok.add(d, c, cor, t)
    ok.metrics()
    bad = d.clone()
    bad[0, 0, 6] = 8.0
    vs = ValStats(8, 10, DEV)
    vs.add(bad, c, cor, t)
    with pytest.raises(RuntimeError, match="class"):
        vs.metrics()
    bad_t = t.clone()
    bad_t[0, 1] = -1.0
    vs = ValStats(8, 10, DEV)
    vs.add(d, c, cor, bad_t)
    with pytest.raises(RuntimeError, match="class"):
        vs.metrics()
