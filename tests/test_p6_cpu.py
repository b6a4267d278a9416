"""The four-level P6 family (models/hub/yolov5{n,s,m,l,x}6.yaml) on the CPU: the generated configurations against the reference's
structure, the fp32 oracle against the reference goldens (tests/golden/make_p6_golden.py), and the stride-64 host geometry."""
import json
import random
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref, tta_ref
from tests.modelgen import build_mirror
from tests.p6gen import ANCHORS_GRID, STRIDES, eval_input, loss_preds, tta_input
from tests.ttagen import pieces
from yolov5_obb_b200 import yolo as Y
from yolov5_obb_b200.engine import tta_geometry
from yolov5_obb_b200.scene import tile_geometry
from yolov5_obb_b200.train_step import multi_scale_max_shape, multi_scale_shape

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))
from check_ref_model_compat import record  # noqa: E402

G = np.load(ROOT / "tests" / "golden" / "p6_golden.npz")


@pytest.mark.parametrize("size", ["n", "s", "m", "l", "x"])
def test_generated_cfg_builds_the_reference_structure(size):
    torch.manual_seed(0)
    for name in (f"yolov5{size}6.yaml", f"yolov5{size}6", f"{size}6"):
        m = Y.Model(name, ch=3, nc=15)
        assert m.yaml_file == f"yolov5{size}6.yaml"
        assert sum(p.numel() for p in m.parameters()) == int(G[f"params/{size}6"])
        det = m.model[-1]
        assert det.nl == 4 and det.na == 3 and m.stride.tolist() == STRIDES
        assert torch.equal(det.anchors, ANCHORS_GRID)
    view = json.loads((ROOT / "tests" / "golden" / "p6_ref_model_view.json").read_text()).get(f"{size}6")
    if view is None:     # the engine view is recorded for n6 / s6 / m6
        return
    torch.manual_seed(0)
    mir = record(Y.Model(f"yolov5{size}6.yaml", ch=3, nc=15))
    assert len(mir["view"]) == len(view["view"])
    for ra, rb in zip(view["view"], mir["view"]):
        assert ra == rb, f"yolov5{size}6: the engine would see\n  reference {ra}\n  mirror    {rb}"
    assert mir["stride"] == view["stride"]
    # same parameter and state_dict names and shapes: a reference checkpoint loads strictly, and the mirror's into the reference
    assert mir["params"] == view["params"]
    assert mir["state_dict"] == view["state_dict"]


def test_p5_names_are_unchanged():
    assert Y.Model("s", nc=15).yaml_file == "yolov5s.yaml" and Y.Model("s", nc=15).model[-1].nl == 3
    for bad in ("yolov5s7.yaml", "q6", "yolov5-p6.yaml"):
        with pytest.raises(FileNotFoundError):
            Y.Model(bad)


def _close(got, want, key, tol=1e-5):
    for k in ("box", "rows"):
        assert np.abs(got[k] - G[f"{key}/{k}"]).max() < tol, (key, k)
    assert np.abs(got["rowsum"] - G[f"{key}/rowsum"]).max() < 200 * tol, key


@pytest.mark.parametrize("size", ["n", "s"])
def test_oracle_reproduces_eval_train_and_tta_goldens(size):
    m = build_mirror(f"{size}6", nc=15, seed=0)
    x = eval_input()
    pred, _ = model_ref.forward(m, x)
    assert pred.shape == (1, 3 * (16 * 24 + 8 * 12 + 4 * 6 + 2 * 3), 200)
    _close(pieces(pred.numpy()), G, f"{size}6/eval")
    raw = model_ref.forward(m, x, training=True)
    assert len(raw) == 4
    for i, r in enumerate(raw):
        assert tuple(r.shape) == tuple(G[f"{size}6/train{i}/shape"])
        _close(pieces(r.detach().reshape(1, -1, 200).numpy()), G, f"{size}6/train{i}", 1e-4)
    m = build_mirror(f"{size}6", nc=15, seed=0)
    aug, _ = tta_ref.forward_augment(m, tta_input())
    _, rows = tta_geometry(256, 320, 64, 4, 3, [8, 16, 32, 64])
    assert tuple(aug.shape) == tuple(G[f"{size}6/tta/shape"]) == (1, rows, 200)
    _close(pieces(aug.numpy()), G, f"{size}6/tta")


def test_oracle_reproduces_the_four_level_loss_golden():
    v = G["loss/hyp"]
    hyp = dict(loss_ref.DEFAULT_HYP, box=float(v[0]), obj=float(v[1]), cls=float(v[2]), theta=float(v[3]),
               anchor_t=float(v[4]), label_smoothing=0.0)
    p = [x.requires_grad_(True) for x in loss_preds(seed=7)]
    tg = torch.from_numpy(G["loss/targets"])
    loss, items = loss_ref.compute_loss(p, tg, ANCHORS_GRID, STRIDES, hyp, 15)
    (loss * 3.0).backward()
    assert abs(loss.item() - float(G["loss/loss"][0])) < 1e-5 * abs(loss.item())
    assert np.abs(items.detach().numpy() - G["loss/items"]).max() < 1e-5
    for i, x in enumerate(p):
        g = x.grad.reshape(-1, 200)
        assert G[f"loss/grows{i}"].size > 0
        assert np.abs(g[:, 4].numpy() - G[f"loss/gobj{i}"]).max() < 1e-9
        assert np.abs(g[G[f"loss/grows{i}"]].numpy() - G[f"loss/gvals{i}"]).max() < 1e-7


def test_tta_geometry_at_stride_64():
    branches, rows = tta_geometry(256, 320, 64, 4, 3, [8, 16, 32, 64])
    assert [(b["h"], b["w"], b["Hp"], b["Wp"]) for b in branches] == [(256, 320, 256, 320), (212, 265, 256, 320),
                                                                       (171, 214, 192, 256)]
    # _clip_augmented drops P6 of the 1.0 branch and P3 of the 0.67 branch
    assert [b["levels"] for b in branches] == [(0, 1, 2), (0, 1, 2, 3), (1, 2, 3)]
    assert rows == int(G["s6/tta/shape"][1])


def test_tile_geometry_rounds_to_the_model_stride():
    assert tile_geometry(1024, 0.5, 64) == (1088, 32, 32.0)
    assert tile_geometry(1024, 0.5) == tile_geometry(1024, 0.5, 32) == (1056, 16, 16.0)
    assert tile_geometry(1024, 0.0, 64) == (1024, 0, 0.0)
    assert tile_geometry(800, 0.5, 64) == (832, 16, 16.0) and tile_geometry(800, 0.5) == (832, 16, 16.0)
    assert tile_geometry(960, 0.5, 64) == (1024, 32, 32.0) and tile_geometry(960, 0.5) == (992, 16, 16.0)


def test_multi_scale_draws_multiples_of_64():
    rng = random.Random(0)
    seen = set()
    for _ in range(2000):
        h, w, _ = multi_scale_shape(1024, 64, 1024, 1024, rng)
        assert h % 64 == 0 and w % 64 == 0 and 512 <= h <= 1536
        seen.add(h)
    assert seen == set(range(512, 1537, 64))
    assert multi_scale_max_shape(1024, 64, 1024, 1024) == (1536, 1536)


def test_train_step_takes_gs_from_the_model():
    from yolov5_obb_b200.train_step import TrainStep
    m = build_mirror("n6", nc=15, seed=0).train()
    ts = TrainStep(m, batch_size=64, imgsz=1024, ema=False)
    assert ts.gs == 64


def _detect_model(nl, na=3):
    anchors = [list(range(10, 10 + 2 * na))] * nl
    det = Y.Detect(nc=15, anchors=anchors, ch=(8,) * nl)
    det.stride = torch.tensor([8.0 * 2 ** i for i in range(nl)])
    m = type("M", (), {})()
    m.hyp, m.model = dict(loss_ref.DEFAULT_HYP), [det]
    return m


def test_compute_loss_levels():
    from yolov5_obb_b200.loss import ComputeLoss, MAX_LEVELS
    assert MAX_LEVELS == 4
    assert ComputeLoss(_detect_model(4)).balance[:4] == [4.0, 1.0, 0.25, 0.06]
    assert ComputeLoss(_detect_model(3)).balance == [4.0, 1.0, 0.4]
    for nl in (2, 5):
        with pytest.raises(RuntimeError, match="3-level .* 4-level"):
            ComputeLoss(_detect_model(nl))
    with pytest.raises(RuntimeError, match="at most 3 anchors"):
        ComputeLoss(_detect_model(4, na=4))
