"""CPU tests of DOTA Task1 evaluation: the CPU restatement oracle/eval_ref.py and the host loaders of
yolov5_obb_b200/dota_eval.py against the reference's own voc_eval / voc_ap / parse_gt (tests/golden/eval_golden.npz)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import eval_ref
from yolov5_obb_b200.dota_eval import load_gt, load_task1

G = np.load(Path(__file__).resolve().parent / "golden" / "eval_golden.npz")
NAMES = [str(n) for n in G["imagenames"]]
CLASSES = [str(c) for c in G["classnames"]]
METRICS = [("voc07", True, 0.5), ("cont", False, 0.5), ("voc07", True, 0.7), ("cont", False, 0.7)]


def write_golden_files(root: Path):
    """The golden's labelTxt and Task1 files under root -> (annopath, detpath) format strings."""
    (root / "labelTxt").mkdir(parents=True, exist_ok=True)
    for k in G.files:
        if k.startswith("labels/"):
            (root / "labelTxt" / f"{k.split('/', 1)[1]}.txt").write_text(str(G[k]))
        elif k.startswith("task1/"):
            (root / f"Task1_{k.split('/', 1)[1]}.txt").write_text(str(G[k]))
    return str(root / "labelTxt" / "{:s}.txt"), str(root / "Task1_{:s}.txt")


def same(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("metric,use07,thr", METRICS)
def test_restatement_matches_reference_voc_eval(metric, use07, thr):
    r = eval_ref.evaluate(G["parse/det_img"], G["parse/det"], G["parse/gt_img"], G["parse/gt"], len(CLASSES), thr, use07)
    key = f"eval/{metric}/{thr}"
    present = G["present"].tolist()
    for c in range(len(CLASSES)):
        if not present[c]:
            continue
        seg = slice(r["class_off"][c], r["class_off"][c + 1])
        assert same(r["rec"][seg], G[f"{key}/rec/{c}"]), (CLASSES[c], "rec")
        assert same(r["prec"][seg], G[f"{key}/prec/{c}"]), (CLASSES[c], "prec")
        assert same(r["ap"][c], G[f"{key}/ap"][c]), (CLASSES[c], "ap")
    assert same(eval_ref.main_map(r["ap"], present), G[f"{key}/map"])


def test_golden_covers_the_edge_classes():
    present = G["present"].tolist()
    ap = G["eval/cont/0.5/ap"]
    assert not present[CLASSES.index("helicopter")]                       # no Task1 file
    assert str(G["task1/harbor"]) == "" and ap[CLASSES.index("harbor")] == 0.0   # empty file
    assert np.isnan(ap[CLASSES.index("roundabout")])                      # detections, no GT
    assert G["eval/voc07/0.5/ap"][CLASSES.index("roundabout")] == 0.0
    assert (G["parse/gt"][:, 1] != 0).any() and (G["parse/gt"][:, 1] == 2).any()


def test_pairwise_sum_is_numpy_add_reduce():
    rng = np.random.default_rng(0)
    for n in list(range(0, 300)) + [1000, 4097, 8191, 8192, 8193, 9001, 16384, 20011, 70001]:
        v = rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 6, n)
        assert same(eval_ref.pairwise_sum(v), np.add.reduce(v)), n


def test_voc07_thresholds_are_multiples_of_a_tenth():
    assert np.arange(0., 1.1, 0.1).tolist() == [k * 0.1 for k in range(11)]


def test_loaders_match_reference_parse(tmp_path):
    annopath, detpath = write_golden_files(tmp_path)
    gt = load_gt(annopath, NAMES, CLASSES, "cpu")
    assert torch.equal(gt.img, torch.from_numpy(G["parse/gt_img"]))
    assert torch.equal(gt.rows, torch.from_numpy(G["parse/gt"]))
    dets = load_task1(detpath, NAMES, CLASSES, "cpu")
    assert torch.equal(dets.img, torch.from_numpy(G["parse/det_img"]))
    assert torch.equal(dets.rows, torch.from_numpy(G["parse/det"]))
    assert dets.present_host == G["present"].tolist()


def test_load_task1_refuses_unknown_image(tmp_path):
    annopath, detpath = write_golden_files(tmp_path)
    with open(detpath.format("ship"), "a") as f:
        f.write("P9999 0.5 1.0 1.0 5.0 1.0 5.0 5.0 1.0 5.0\n")
    with pytest.raises(RuntimeError, match="P9999"):
        load_task1(detpath, NAMES, CLASSES, "cpu")


def test_load_gt_refuses_object_line_with_more_than_10_fields(tmp_path):
    """parse_gt sets `difficult` only for 9 or 10 fields, and voc_eval then fails with a KeyError: refused at load time."""
    (tmp_path / "A.txt").write_text("gsd:0.5\n1 1 5 1 5 5 1 5 ship 0\n1 1 5 1 5 5 1 5 ship 0 extra\n")
    with pytest.raises(RuntimeError, match="extra"):
        load_gt(str(tmp_path / "{:s}.txt"), ["A"], ["ship"], "cpu")
    gt = load_gt(str(tmp_path / "{:s}.txt"), ["A"], ["plane"], "cpu")   # a class outside classnames is ignored, as before
    assert gt.rows.shape == (0, 10)
