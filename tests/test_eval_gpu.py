"""GPU tests of DOTA Task1 evaluation (yolov5_obb_b200/dota_eval.py, csrc/dota_eval.cu): the reference's own voc_eval / voc_ap
results (tests/golden/eval_golden.npz), the CPU restatement oracle/eval_ref.py on tie-heavy inputs at scale and on edge cases,
the in-memory route against the Task1 file route, and the refusals."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import eval_ref
from tests.scenegen import tile_rows
from tests.test_eval_cpu import CLASSES, G, METRICS, NAMES, write_golden_files
from yolov5_obb_b200.dota_eval import GroundTruth, Task1Detections, evaluate_task1, load_gt, load_task1
from yolov5_obb_b200.scene import merge_tiles

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def same(a, b):
    a = torch.as_tensor(a, dtype=torch.float64).cpu()
    b = torch.as_tensor(b, dtype=torch.float64).cpu()
    return a.shape == b.shape and torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(0.0), b.nan_to_num(0.0))


def device_eval(det_img, det10, gt_img, gt10, names, nc, thr, use07):
    dets = Task1Detections(names, nc, DEV).add_rows(torch.as_tensor(det_img, dtype=torch.int32).to(DEV),
                                                    torch.as_tensor(det10, dtype=torch.float64).reshape(-1, 10).to(DEV))
    gt = GroundTruth(torch.as_tensor(gt_img, dtype=torch.int32).to(DEV),
                     torch.as_tensor(gt10, dtype=torch.float64).reshape(-1, 10).to(DEV), names, nc)
    return evaluate_task1(dets, gt, thr, use07)


def assert_equals_restatement(res, want, nc):
    assert torch.equal(res.class_off.cpu(), torch.from_numpy(want["class_off"]))
    assert torch.equal(res.npos.cpu(), torch.from_numpy(want["npos"]))
    assert same(res._rec, want["rec"]) and same(res._prec, want["prec"])
    assert same(res.ap, want["ap"])


@pytest.mark.parametrize("metric,use07,thr", METRICS)
def test_equals_reference_voc_eval_on_golden(tmp_path, metric, use07, thr):
    annopath, detpath = write_golden_files(tmp_path)
    res = evaluate_task1(load_task1(detpath, NAMES, CLASSES, DEV), load_gt(annopath, NAMES, CLASSES, DEV), thr, use07)
    key = f"eval/{metric}/{thr}"
    for c in range(len(CLASSES)):
        if G["present"][c]:
            assert same(res.rec(c), G[f"{key}/rec/{c}"]), CLASSES[c]
            assert same(res.prec(c), G[f"{key}/prec/{c}"]), CLASSES[c]
            assert same(res.ap[c], G[f"{key}/ap"][c]), CLASSES[c]
    assert torch.equal(res.present.cpu(), torch.from_numpy(G["present"]))
    assert same(res.map, G[f"{key}/map"])


def _rects(rng, n, W=1000.0):
    cx, cy = rng.uniform(20, W - 20, n), rng.uniform(20, W - 20, n)
    l, s = rng.uniform(8, 40, n), rng.uniform(6, 20, n)
    th = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(-np.pi / 2, np.pi / 2, n))
    c, si = np.cos(th), np.sin(th)
    pts = [np.stack([cx + dx * c - dy * si, cy + dx * si + dy * c], 1) for dx, dy in ((-l, -s), (l, -s), (l, s), (-l, s))]
    return np.round(np.concatenate(pts, 1), 1)


def tie_heavy_set(seed, n_images=24, nc=15, big=14000):
    """GTs (class 0 has `big` of them, about 10 % difficult) and Task1-rounded detections: most GTs detected once or twice
    with jitter, plus false positives; scores round(u, 2) so that ties are everywhere."""
    rng = np.random.default_rng(seed)
    gt_img, gt = [], []
    counts = [big] + [int(rng.integers(20, 200)) for _ in range(nc - 1)]
    for c, n in enumerate(counts):
        img = rng.integers(0, n_images, n)
        diff = (rng.random(n) < 0.1).astype(np.float64)
        gt_img.append(img)
        gt.append(np.concatenate([np.full((n, 1), float(c)), diff[:, None], _rects(rng, n)], 1))
    gt_img, gt = np.concatenate(gt_img), np.concatenate(gt)
    reps = rng.choice([0, 1, 1, 1, 1, 2], len(gt))
    src = np.repeat(np.arange(len(gt)), reps)
    jit = np.round(gt[src, 2:] + rng.normal(0, 0.5, (len(src), 1)) + rng.normal(0, 0.3, (len(src), 8)), 1)
    n_fp = len(src) // 5
    fp = _rects(rng, n_fp)
    det = np.concatenate([np.concatenate([gt[src, :1], np.zeros((len(src), 1)), jit], 1),
                          np.concatenate([rng.integers(0, nc, (n_fp, 1)).astype(np.float64), np.zeros((n_fp, 1)), fp], 1)])
    det_img = np.concatenate([gt_img[src], rng.integers(0, n_images, n_fp)])
    det[:, 1] = np.round(rng.uniform(0.01, 1.0, len(det)), 2)
    perm = rng.permutation(len(det))
    return det_img[perm], det[perm], gt_img, gt, n_images, nc


@pytest.fixture(scope="module")
def tie_set():
    return tie_heavy_set(11)


@pytest.mark.parametrize("use07,thr", [(True, 0.5), (False, 0.5), (False, 0.7)])
def test_equals_restatement_on_tie_heavy_set_at_scale(tie_set, use07, thr):
    det_img, det, gt_img, gt, n_images, nc = tie_set
    want = eval_ref.evaluate(det_img, det, gt_img, gt, nc, thr, use07)
    steps = np.count_nonzero(np.diff(np.concatenate([[0.0], want["rec"][:want["class_off"][1]]])))
    assert steps > 8192 and len(np.unique(det[:, 1])) <= 100
    res = device_eval(det_img, det, gt_img, gt, [f"I{i}" for i in range(n_images)], nc, thr, use07)
    assert_equals_restatement(res, want, nc)
    assert same(res.map, eval_ref.main_map(want["ap"], [True] * nc))


def test_edge_cases_follow_restatement():
    """Zero-area polygons (NaN IoU: a false positive), a detection in an image without a GT of its class, a match to a
    difficult GT (neither TP nor FP), a second match to a taken GT (FP), and a class with detections but no GT."""
    sq = [10.0, 10.0, 50.0, 10.0, 50.0, 50.0, 10.0, 50.0]
    flat = [100.0, 100.0, 120.0, 100.0, 120.0, 100.0, 100.0, 100.0]
    gt = np.array([[0, 0] + sq, [0, 1] + [x + 200 for x in sq], [0, 0] + flat, [1, 0] + sq], np.float64)
    gt_img = np.array([0, 0, 0, 1])
    det = np.array([[0, 0.9] + sq, [0, 0.9] + sq, [0, 0.8] + [x + 200 for x in sq], [0, 0.7] + flat, [0, 0.6] + sq,
                    [1, 0.5] + sq, [2, 0.4] + sq], np.float64)
    det_img = np.array([0, 0, 0, 0, 1, 1, 0])
    for use07 in (True, False):
        want = eval_ref.evaluate(det_img, det, gt_img, gt, 3, 0.5, use07)
        res = device_eval(det_img, det, gt_img, gt, ["A", "B"], 3, 0.5, use07)
        assert_equals_restatement(res, want, 3)
    # class 0, sorted: TP, FP (taken), ignored (difficult), FP (NaN IoU), FP (no GT of class 0 in image B)
    assert want["rec"][:5].tolist() == [0.5, 0.5, 0.5, 0.5, 0.5]
    assert want["prec"][:5].tolist() == [1.0, 0.5, 0.5, 1 / 3, 0.25]
    assert np.isnan(want["ap"][2]) and want["npos"].tolist() == [2, 1, 0]


def test_in_memory_route_equals_task1_file_route(tmp_path):
    GS = np.load(Path(__file__).resolve().parent / "golden" / "scene_golden.npz")
    names = [str(n) for n in GS["merge/names"]][:15]
    scenes = [merge_tiles(torch.from_numpy(GS["merge/rows"]).to(DEV), torch.from_numpy(GS["merge/counts"]).to(DEV),
                          torch.from_numpy(GS["merge/origins"]).to(DEV), 15, 16.0, 0.2)]
    origins, rows, counts = tile_rows(2400, 1800, 300, nc=15, seed=9)
    scenes.append(merge_tiles(torch.from_numpy(rows).to(DEV), torch.from_numpy(counts).to(DEV),
                              torch.from_numpy(origins).to(DEV), 15, 16.0, 0.2))
    imagenames = ["P0000", "P0001"]
    rng = np.random.default_rng(4)
    (tmp_path / "labelTxt").mkdir()
    for i, sc in enumerate(scenes):
        r = sc.rows.cpu().numpy()
        keep = r[rng.random(len(r)) < 0.7]
        lines = ["imagesource:GoogleEarth", "gsd:0.5"]
        for row in keep:
            poly = np.round(row[2:] + rng.normal(0, 1.5, 8), 1)
            lines.append(" ".join(map(str, poly.tolist())) + f" {names[int(row[0])]} {int(rng.random() < 0.1)}")
        (tmp_path / "labelTxt" / f"{imagenames[i]}.txt").write_text("\n".join(lines) + "\n")
        sc.write_task1(tmp_path / "task1", imagenames[i], names)
    gt = load_gt(str(tmp_path / "labelTxt" / "{:s}.txt"), imagenames, names, DEV)
    mem = Task1Detections(imagenames, 15, DEV)
    for i, sc in enumerate(scenes):
        mem.add(i, sc)
    files = load_task1(str(tmp_path / "task1" / "Task1_{:s}.txt"), imagenames, names, DEV)
    # scene-major in memory, class-major from the files: the same rows in the same order within every class
    assert mem.rows.shape == files.rows.shape
    for c in range(15):
        a, b = mem.rows[:, 0] == c, files.rows[:, 0] == c
        assert torch.equal(mem.rows[a], files.rows[b]) and torch.equal(mem.img[a], files.img[b])
    for use07 in (True, False):
        a, b = evaluate_task1(mem, gt, 0.5, use07), evaluate_task1(files, gt, 0.5, use07)
        assert same(a._rec, b._rec) and same(a._prec, b._prec) and same(a.ap, b.ap)
        assert torch.equal(a.present, b.present) and same(a.map, b.map)
        assert a.map > 0.1


def test_refusals(tmp_path):
    det_img, det = torch.zeros(2, dtype=torch.int32), torch.zeros((2, 10), dtype=torch.float64)
    det[:, 2:] = torch.tensor([0.0, 0.0, 4.0, 0.0, 4.0, 4.0, 0.0, 4.0], dtype=torch.float64)
    gt = GroundTruth(det_img.to(DEV), det.to(DEV), ["A"], 2)
    with pytest.raises(RuntimeError):   # CPU tensors
        evaluate_task1(Task1Detections(["A"], 2, "cpu").add_rows(det_img, det), gt)
    with pytest.raises(RuntimeError):   # wrong dtype
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img.to(DEV), det.float().to(DEV)), gt)
    with pytest.raises(RuntimeError):   # wrong shape
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img.to(DEV), det[:, :9].contiguous().to(DEV)), gt)
    with pytest.raises(RuntimeError):   # img of another length
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img[:1].to(DEV), det.to(DEV)), gt)
    ok = evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img.to(DEV), det.to(DEV)), gt)
    want = eval_ref.evaluate(det_img.numpy(), det.numpy(), det_img.numpy(), det.numpy(), 2)
    assert same(ok.map, eval_ref.main_map(want["ap"], [True, False]))
    bad_cls = det.clone()
    bad_cls[1, 0] = 2.0
    with pytest.raises(RuntimeError, match="class"):
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img.to(DEV), bad_cls.to(DEV)), gt).map
    bad_img = torch.tensor([0, 1], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="image"):
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(bad_img.to(DEV), det.to(DEV)), gt).check()
    with pytest.raises(RuntimeError, match="class"):
        evaluate_task1(Task1Detections(["A"], 2, DEV).add_rows(det_img.to(DEV), det.to(DEV)),
                       GroundTruth(det_img.to(DEV), bad_cls.to(DEV), ["A"], 2)).map
    (tmp_path / "Task1_x.txt").write_text("B 0.5 0 0 4 0 4 4 0 4\n")
    with pytest.raises(RuntimeError, match="'B'"):
        load_task1(str(tmp_path / "Task1_{:s}.txt"), ["A"], ["x"], DEV)


def test_in_memory_route_on_the_default_device(tmp_path):
    """Task1Detections / load_gt / load_task1 with their default device ("cuda", no index) and SceneDetections made on the
    current device: the scene -> detections -> mAP loop as INTEGRATION.md writes it."""
    GS = np.load(Path(__file__).resolve().parent / "golden" / "scene_golden.npz")
    names = [str(n) for n in GS["merge/names"]][:15]
    sc = merge_tiles(torch.from_numpy(GS["merge/rows"]).to(DEV), torch.from_numpy(GS["merge/counts"]).to(DEV),
                     torch.from_numpy(GS["merge/origins"]).to(DEV), 15, 16.0, 0.2)
    r = sc.rows.cpu().numpy()
    (tmp_path / "labelTxt").mkdir()
    lines = [" ".join(map(str, row[2:].tolist())) + f" {names[int(row[0])]} 0" for row in r[::2]]
    (tmp_path / "labelTxt" / "P0000.txt").write_text("\n".join(lines) + "\n")
    sc.write_task1(tmp_path / "task1", "P0000", names)
    with torch.cuda.device(DEV):
        gt = load_gt(str(tmp_path / "labelTxt" / "{:s}.txt"), ["P0000"], names)
        mem = Task1Detections(["P0000"], len(names)).add(0, sc)
        files = load_task1(str(tmp_path / "task1" / "Task1_{:s}.txt"), ["P0000"], names)
    assert mem.device == torch.device(DEV) and mem.rows.device == torch.device(DEV)
    a, b = evaluate_task1(mem, gt), evaluate_task1(files, gt)
    assert same(a.ap, b.ap) and same(a.map, b.map) and a.map > 0.3
