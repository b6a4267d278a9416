"""GPU tests of model ensembles (yolov5_obb_b200.ensemble.Ensemble, engine.EnsemblePlan):
  * the rows are bit-equal to torch.cat of the members' own forward (and forward_augment) outputs;
  * the whole output against the REFERENCE's models/experimental.Ensemble golden (yolov5n + yolov5n6);
  * records + NMS equal tensor + NMS, and the NMS keep sets equal the oracle NMS on the engine's own rows;
  * the image is staged once per batch, and resampled once per (TTA scale, member gs);
  * DetectPipeline (two slots, run_images with a P6 member), Validator (tensor, raw and augment=True forms) and
    SceneDetector (1088^2 tiles with a P6 member) against compositions of the public calls;
  * the re-plan after an in-place update of one member;
  * the conv configurations the ensembles add (1088^2 P5 plans, P5 test-time augmentation at multiples of 64) are reached
    by the exact launch checks (tests/test_conv_plans_wide_gpu.census)."""
import copy
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle.postprocess import non_max_suppression_obb as oracle_nms
from tests.ensemblegen import DET_KW, MEMBERS, NC, NMS_KW, ensemble_input
from tests.modelgen import build_mirror
from tests.recordcheck import check_records
from tests.test_engine_gpu import _compare
from tests.ttagen import pieces
from yolov5_obb_b200 import general
from yolov5_obb_b200.ensemble import Ensemble, attempt_load

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
DEV = "cuda:0"


def _members(keys, seed=0, **kw):
    return [build_mirror(k, nc=NC, seed=seed + i, **kw).to(DEV) for i, k in enumerate(keys)]


def _x(B, H, W, seed, u8=False):
    g = torch.Generator().manual_seed(seed)
    if u8:
        return torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8).to(DEV)
    return torch.rand(B, 3, H, W, generator=g).to(DEV)


# ---- rows ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keys,B,H,W", [(("s", "m"), 2, 256, 320), (("s", "s6"), 2, 256, 320),
                                        (("n6", "s", "n"), 1, 192, 384), (("s", "s6"), 1, 1024, 1024)])
def test_rows_equal_cat_of_members(keys, B, H, W):
    members = _members(keys)
    ens = attempt_load(members)
    for u8 in (False, True):
        x = _x(B, H, W, len(keys) + H, u8)
        got = ens(x)[0].clone()
        want = torch.cat([m(x)[0] for m in members], 1)
        assert torch.equal(got, want), (keys, u8)
        got = ens(x, augment=True)[0].clone()
        want = torch.cat([m.forward_augment(x)[0] for m in members], 1)
        assert torch.equal(got, want), (keys, u8, "augment")
        assert torch.equal(ens.forward_augment(x)[0], want)
    plan = ens.records_plan((B, 3, H, W), DEV)
    assert plan.row_bases == [0] + list(np.cumsum([m(x)[0].shape[1] for m in members])[:-1])


# ---- the reference golden -----------------------------------------------------------------------------------------------
def _golden_nms_agreement(got, ref):
    """Fraction of the reference's kept rows with a kept row of the same class whose centre lies within 1 px and whose
    confidence is within 2e-2."""
    if ref.shape[0] == 0:
        return 1.0
    g = torch.from_numpy(got) if isinstance(got, np.ndarray) else got.cpu()
    r = torch.from_numpy(ref)
    close = ((g[None, :, :2] - r[:, None, :2]).abs().amax(-1) <= 1.0) & (g[None, :, 6] == r[:, None, 6]) & \
        ((g[None, :, 5] - r[:, None, 5]).abs() <= 2e-2)
    return close.any(1).float().mean().item()


@pytest.mark.parametrize("form", ["plain", "tta"])
def test_matches_reference_golden(form):
    G = np.load(ROOT / "tests" / "golden" / "ensemble_golden.npz")
    ens = Ensemble([build_mirror(k, nc=NC, seed=0, **DET_KW).to(DEV) for k in MEMBERS])   # (every member from seed 0)
    x = ensemble_input()
    assert x.double().sum().item() == float(G["x_sum"])
    pred, none = ens(x.to(DEV), augment=form == "tta")
    torch.cuda.synchronize()
    assert none is None and tuple(pred.shape) == tuple(G[f"{form}/shape"])
    got = pieces(pred.cpu().numpy())
    _compare(torch.from_numpy(got["rows"]), torch.from_numpy(G[f"{form}/rows"]), f"ensemble {form} sampled rows vs golden")
    box, ref = torch.from_numpy(got["box"]), torch.from_numpy(G[f"{form}/box"])
    frac_bad = ((box - ref).abs() > ref.abs() * 3e-2 + 3e-2).float().mean().item()
    print(f"ensemble {form} boxes vs golden: max err {(box - ref).abs().max().item():.4g}, out-of-tol {frac_bad:.2e}")
    assert frac_bad < 1e-3
    # the reference NMS on the reference rows.  The scores of these random-weight members sit in a narrow band of thousands
    # of overlapping candidates, so which rows survive moves with any rounding (an fp32 perturbation of 4e-3 keeps under
    # half of them): only the kept count is compared here, and the keep sets are checked exactly against the oracle NMS on
    # the engine's own rows (test_records_plus_nms_equal_tensor_plus_nms_and_oracle)
    dets = general.non_max_suppression_obb(pred, **NMS_KW)
    for b, d in enumerate(dets):
        ref_d = G[f"{form}/nms/{b}"]
        print(f"ensemble {form} image {b}: {d.shape[0]} kept, reference {ref_d.shape[0]}, "
              f"{_golden_nms_agreement(d, ref_d):.3f} of the reference's matched")
        assert d.shape[0] == ref_d.shape[0] and d.shape[1] == 7


# ---- records + NMS ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("augment", [False, True])
def test_records_plus_nms_equal_tensor_plus_nms_and_oracle(augment):
    ens = Ensemble(_members(("n", "s6"), seed=3, **DET_KW))
    x = _x(2, 256, 320, 5)
    pred = ens(x, augment=augment)[0].clone()
    rec = ens.detect_records(x, augment=augment)
    assert rec.data.shape == (2, pred.shape[1], 24) and rec.nc == NC
    patched, near_ties = check_records(pred, rec.data, NC)
    assert near_ties <= max(2, pred.shape[0] * pred.shape[1] // 1000)
    for kw in (dict(conf_thres=0.3, iou_thres=0.45, multi_label=True, max_det=300),
               dict(conf_thres=0.3, iou_thres=0.45, multi_label=False, max_det=100)):
        a = general.non_max_suppression_obb(patched, **kw)
        b = general.non_max_suppression_obb(rec, **kw)
        o = oracle_nms(patched.cpu(), nms_mode=1, **kw)
        assert sum(t.shape[0] for t in a) > 0
        for u, v, w in zip(a, b, o):
            assert torch.equal(u, v)
            g, e = u.cpu().numpy(), w.numpy()
            assert g.shape == e.shape, (g.shape, e.shape)
            # (a decisive IoU within FMA distance of the threshold may flip one box, as in test_postprocess_gpu)
            assert np.array_equal(g, e) or (g == e).all(1).mean() > 0.995


# ---- the staged input ---------------------------------------------------------------------------------------------------
def test_one_staged_input_and_one_resample_per_scale_and_gs():
    ens = Ensemble(_members(("n", "n6", "s")))
    B, H, W = 2, 256, 320
    plain = ens.records_plan((B, 3, H, W), DEV)
    labels = [s[0] for s in plain.steps]
    assert labels == [("stem",), ("layers", 0, 0), ("layers", 1, 0), ("layers", 2, 0)]
    assert all(e.x_s2d is plain.x_s2d for e in plain.members)
    tta = ens.tta_plan((B, 3, H, W), DEV)
    labels = [s[0] for s in tta.steps]
    assert labels.count(("stem",)) == 1
    assert sorted(l[1:] for l in labels if l[0] == "resample") == [(1, 32), (1, 64), (2, 32), (2, 64)]
    assert sorted(l[1:] for l in labels if l[0] == "layers") == [(i, k) for i in range(3) for k in range(3)]
    for k in range(3):
        xs = [p.engines[k].x_s2d for p in tta.members]
        assert xs[0] is xs[2] and (xs[0] is xs[1]) == (k == 0)   # n and s share gs 32; n6 has gs 64; scale 1 is shared
    # the one staged input really is what every member reads: the member rows equal their own plans' on a second call
    x = _x(B, H, W, 9)
    got = ens.detect_records(x).data.clone()
    for m, base in zip(ens, plain.row_bases):
        own = m.detect_records(x).data
        assert torch.equal(got[:, base:base + own.shape[1]], own)


# ---- callers ------------------------------------------------------------------------------------------------------------
def test_detect_pipeline_two_slots_and_run_images_with_a_p6_member():
    from tests import letterboxgen as LG
    from tests.test_letterbox_gpu import KW, R, P, _existing_path
    from tests.tilegen import synth_tiles
    from yolov5_obb_b200.pipeline import DetectPipeline
    ens = Ensemble(_members(("n", "n6"), **DET_KW))
    kw = dict(conf_thres=0.3, iou_thres=0.45, multi_label=True, max_det=300)
    batches = [synth_tiles(2, 256, seed=s).pin_memory() for s in range(1, 8)]
    want = [[d.cpu() for d in general.non_max_suppression_obb(ens.detect_records(xb.to(DEV)), **kw)] for xb in batches]
    pipe = DetectPipeline(ens, 0.3, 0.45, 300, multi_label=True, device=DEV, slots=2)
    assert pipe.slots == 2 and pipe.fused
    got = list(pipe(iter(batches)))
    assert len(got) == len(want) and sum(d.shape[0] for w in want for d in w) > 0
    for g, w in zip(got, want):
        assert all(torch.equal(a, b) for a, b in zip(g, w)) and len(g) == len(w)
    # decoded images of odd sizes, letterboxed to multiples of the ensemble's stride 64
    sizes = [(300, 400), (97, 211), (200, 140), (260, 250)]
    images = [LG.synth_image(h, w, 80 + i) for i, (h, w) in enumerate(sizes)]
    want = []
    for im in images:
        lbx = R.to_chw_rgb(R.letterbox(im, 256, auto=True, stride=64)[0])[None]
        assert lbx.shape[2] % 64 == 0 and lbx.shape[3] % 64 == 0
        want += _existing_path(ens, lbx, [P.detect_pad_gain(lbx.shape[2:], im.shape[:2])])
    pipe = DetectPipeline(ens, multi_label=True, device=DEV, slots=2, **KW)
    got = list(pipe.run_images(iter(images), img_size=256, auto=True))
    assert len(got) == len(images) and sum(w[1].shape[0] for w in want) > 0
    for g, (poly, rows) in zip(got, want):
        assert torch.equal(g.rows, rows) and torch.equal(g.polys, poly)


def _val_ensemble():
    from tests.modelgen import calibrated_bench_model
    return Ensemble([calibrated_bench_model("n", conf=0.1).to(DEV), calibrated_bench_model("n6", conf=0.1).to(DEV)])


def test_validator_tensor_augment_and_raw_forms():
    from tests.test_tta_gpu import _tta_composition
    from tests.test_valmetrics_gpu import _composition, _loader, _model_and_batches, assert_same
    from yolov5_obb_b200.val import Validator
    ens = _val_ensemble()
    _, batches = _model_and_batches()
    assert all(b.shape[2] % 64 == 0 and b.shape[3] % 64 == 0 for b in batches)
    loader = _loader(ens, batches, 0.1)
    v = Validator(ens, conf_thres=0.1, iou_thres=0.4, max_det=300)
    m = v(loader)
    assert_same(m, _composition(ens, loader, v.nms, v.iouv.cpu(), ens.nc))
    assert m.seen == sum(b.shape[0] for b in batches) and v.reruns == 0 and m.results[2] > 0
    va = Validator(ens, conf_thres=0.1, iou_thres=0.4, max_det=300, augment=True)
    ma = va(loader)
    assert_same(ma, _tta_composition(ens, loader, va.nms, va.iouv.cpu(), ens.nc))
    assert not np.array_equal(np.array(ma.results), np.array(m.results))


def test_validator_raw_form_equals_tensor_form():
    from tests import letterboxgen as LG
    from tests.test_letterbox_gpu import P, _oracle_rect
    from yolov5_obb_b200.rboxs_utils import poly2rbox
    from yolov5_obb_b200.val import Validator
    ens = Ensemble(_members(("n", "n6"), **DET_KW))
    sizes = [(300, 400), (256, 256), (97, 211), (200, 140), (260, 250)]
    images = [LG.synth_image(h, w, 90 + i) for i, (h, w) in enumerate(sizes)]
    img_size, bs = 256, 2
    order, shapes = P.rect_batch_shapes([(im.shape[1], im.shape[0]) for im in images], bs, img_size, 64, 0.5)
    raw, tens = [], []
    for b in range(len(shapes)):
        idx = [int(k) for k in order[b * bs:(b + 1) * bs]]
        places = [P.place_rect(images[k].shape[0], images[k].shape[1], img_size, shapes[b]) for k in idx]
        tg = []
        for j, (k, p) in enumerate(zip(idx, places)):
            polys = p.map_labels(LG.synth_polys(images[k].shape[0], images[k].shape[1], 4, 900 + k))
            rb = poly2rbox(torch.from_numpy(polys).float().to(DEV), use_pi=True).float().cpu()
            tg.append(torch.cat([torch.full((4, 1), float(j)), torch.full((4, 1), float(k % 15)), rb], 1))
        targets = torch.cat(tg)
        sh = [p.shapes for p in places]
        raw.append(([images[k] for k in idx], targets, None, sh))
        tens.append((torch.from_numpy(_oracle_rect([images[k] for k in idx], img_size, shapes[b])), targets, None, sh))
    a = Validator(ens, max_det=300)(raw)
    b = Validator(ens, max_det=300)(tens)
    assert a.seen == b.seen == len(images)
    assert a.results == b.results and np.array_equal(a.maps, b.maps) and np.array_equal(a.nt, b.nt)
    assert np.array_equal(a.ap_full, b.ap_full) and np.array_equal(a.p_curve, b.p_curve)


def test_scene_detector_with_a_p6_member_uses_1088_tiles():
    from tests.test_scene_gpu import _scene, _torch_tiles
    from yolov5_obb_b200.scene import SceneDetector, merge_tiles, split_origins
    ens = Ensemble(_members(("n", "n6"), **DET_KW))
    det = SceneDetector(ens, batch_size=3, conf_thres=0.3)
    assert (det.size, det.border, det.pad_xy) == (1088, 32, 32.0)
    scene = _scene(1200, 1500, 4)
    origins = split_origins(1200, 1500)
    assert len(origins) == 4
    got = det.det(scene.to(DEV)).rows.cpu()
    assert det.model.records_plan((3, 3, 1088, 1088), DEV).rows_total == sum(
        3 * sum((1088 // int(s)) ** 2 for s in m.stride) for m in ens)
    # the composition: torch-built tiles -> the ensemble's records -> NMS -> merge
    tiles = _torch_tiles(scene, origins, 1024, 1088, 32).to(DEV)
    packed, counts = general.non_max_suppression_obb(ens.detect_records(tiles), 0.3, 0.4, multi_label=True, max_det=1500,
                                                     return_packed=True)
    org = torch.tensor(origins, dtype=torch.int32, device=DEV)
    want = merge_tiles(packed, torch.tensor(counts, dtype=torch.int64, device=DEV), org, NC, 32.0, 0.2).rows.cpu()
    assert sum(counts) > 100 and want.shape[0] > 10
    assert torch.equal(got, want)


# ---- re-plan ------------------------------------------------------------------------------------------------------------
def test_replan_after_member_update():
    members = _members(("s", "n6"), seed=2)
    ens = Ensemble(members)
    x = _x(2, 256, 320, 4)
    before = ens(x)[0].clone()
    before_aug = ens(x, augment=True)[0].clone()
    ens.detect_records(x)
    with torch.no_grad():
        members[1].model[-1].m[2].bias.add_(0.25)
        members[1].model[4].cv1.bn.weight.mul_(1.1)
    after = ens(x)[0].clone()
    assert not torch.equal(before, after)
    fresh = Ensemble([copy.deepcopy(m) for m in members])
    assert torch.equal(after, fresh(x)[0])
    after_aug = ens(x, augment=True)[0].clone()
    assert not torch.equal(before_aug, after_aug) and torch.equal(after_aug, fresh(x, augment=True)[0])
    assert torch.equal(ens.detect_records(x).data, fresh.detect_records(x).data)
    # the first member's rows did not move
    r0 = members[0](x)[0].shape[1]
    assert torch.equal(before[:, :r0], after[:, :r0])


def test_refusals_on_device():
    ens = Ensemble(_members(("n", "n6")))
    with pytest.raises(RuntimeError, match="largest stride 64"):
        ens(torch.zeros(1, 3, 224, 320, device=DEV))
    with pytest.raises(RuntimeError):
        ens(torch.zeros(1, 3, 256, 320))                                 # host tensor
    with pytest.raises(RuntimeError, match="plain ensemble plan"):
        ens.tta_plan((1, 3, 256, 320), DEV).forward_s2d()
    with pytest.raises(RuntimeError, match="different devices"):
        Ensemble([build_mirror("n", nc=NC).to(DEV), build_mirror("n", nc=NC)])


# ---- conv configurations ------------------------------------------------------------------------------------------------
# the plans ensembles add for P5 members: 1088^2 records plans (scene tiles and val.py's rect shapes once a P6 member sets
# the stride to 64) and test-time augmentation of a 1088^2 input
ENSEMBLE_PLANS = [("s", 16, 1088, 1088, "records"), ("x", 16, 1088, 1088, "records"),
                  ("s", 16, 1088, 1088, "tta"), ("s", 16, 1088, 1088, "tta-records"),
                  ("m", 16, 1088, 1088, "tta"), ("m", 16, 1088, 1088, "tta-records")]


def test_ensemble_plans_reach_only_checked_configurations():
    from tests import test_conv_plans_wide_gpu as CW
    missing = CW._measured("ensemble census", CW.census, CW.CHECKED, ENSEMBLE_PLANS)
    assert not missing, f"{len(missing)} configurations of ensemble plans no exact check runs: " + \
        "; ".join(f"{CW.key_str(k)} ({p} {i})" for k, (p, i) in missing.items())
