"""Golden vectors of the four-level P6 family from the REFERENCE (models/hub/yolov5{n,s,m,l,x}6.yaml, models/yolo.py Model,
utils/loss.py ComputeLoss with the clamp shim of make_loss_golden.py) — run in the authoring container:
    python tests/golden/make_p6_golden.py
Writes p6_golden.npz and p6_ref_model_view.json:
  for yolov5n6 and yolov5s6 (nc=15, torch seed 0, tests/modelgen.seeded_state):
    eval/*    the eval output on tests/p6gen.eval_input(), stored as tests/ttagen.pieces() describes;
    train/*   the train-mode Detect logits on the same image (batch-statistic BatchNorm), per level [1, 3, H, W, 200] pieces;
    tta/*     `m(x, augment=True)` on tests/p6gen.tta_input(), as pieces;
  loss/*      ComputeLoss (nl = 4, balance 4.0 / 1.0 / 0.25 / 0.06) on tests/p6gen.loss_preds() and loss_targets() with the
              hyp train.py gives a 4-level model: loss, items and the gradients of (loss * 3) as make_loss_golden.py stores them;
  params/<k>  the parameter count of yolov5<k>.yaml for all five scales;
and, as check_ref_model_compat.py does for P5, the engine's view of the reference Model for n6 / s6 / m6."""
import json
import sys
import types
from pathlib import Path

import numpy as np
import torch
import yaml

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
from models.yolo import Model  # noqa: E402  (the reference)
from check_ref_model_compat import record  # noqa: E402
from oracle.loss_ref import scaled_hyp  # noqa: E402
from tests.modelgen import seeded_state  # noqa: E402
from tests.p6gen import eval_input, loss_preds, loss_targets, tta_input, LOSS_W  # noqa: E402
from tests.ttagen import pieces  # noqa: E402

src = (ref_import.REF / "utils" / "loss.py").read_text()
src = src.replace("gj.clamp_(0, feature_wh[1] - 1), gi.clamp_(0, feature_wh[0] - 1)",
                  "gj.clamp_(0, int(feature_wh[1]) - 1), gi.clamp_(0, int(feature_wh[0]) - 1)")
assert "int(feature_wh[1])" in src
ref_loss = types.ModuleType("ref_loss")
ref_loss.__dict__["__name__"] = "utils.loss_shimmed"
exec(compile(src, str(ref_import.REF / "utils" / "loss.py"), "exec"), ref_loss.__dict__)


def ref_model(size):
    torch.manual_seed(0)
    return Model(f"models/hub/yolov5{size}6.yaml", ch=3, nc=15)


def main():
    out, view = {}, {}
    for size in ("n", "s", "m", "l", "x"):
        m = ref_model(size)
        out[f"params/{size}6"] = np.int64(sum(p.numel() for p in m.parameters()))
        if size in ("n", "s", "m"):
            view[f"{size}6"] = record(m)
        if size not in ("n", "s"):
            continue
        seeded_state(m, 0).eval()
        x = eval_input()
        with torch.no_grad():
            pred, _ = m(x)
            for k, v in pieces(pred.numpy()).items():
                out[f"{size}6/eval/{k}"] = v
            aug, _ = m(tta_input(), augment=True)
            for k, v in pieces(aug.numpy()).items():
                out[f"{size}6/tta/{k}"] = v
            out[f"{size}6/tta/shape"] = np.array(aug.shape)
            m.train()
            raw = m(x)
            for i, r in enumerate(raw):
                flat = r.reshape(1, -1, r.shape[-1]).numpy()
                for k, v in pieces(flat).items():
                    out[f"{size}6/train{i}/{k}"] = v
                out[f"{size}6/train{i}/shape"] = np.array(r.shape)
        print(f"yolov5{size}6: {int(out[f'params/{size}6'])} parameters, eval {tuple(pred.shape)}, tta {tuple(aug.shape)}, "
              f"train {[tuple(r.shape) for r in raw]}")

    hyp = yaml.safe_load((ref_import.REF / "data" / "hyps" / "obb" / "hyp.finetune_dota.yaml").read_text())
    h = scaled_hyp(hyp, 4, 15, LOSS_W)
    m = ref_model("n")
    m.hyp = h
    cl = ref_loss.ComputeLoss(m)
    assert list(cl.balance[:4]) == [4.0, 1.0, 0.25, 0.06]
    p = [x.requires_grad_(True) for x in loss_preds(seed=7)]
    tg = loss_targets(seed=7)
    loss, items = cl(p, tg)
    (loss * 3.0).backward()
    out["loss/targets"] = tg.numpy()
    out["loss/loss"] = loss.detach().numpy()
    out["loss/items"] = items.numpy()
    out["loss/hyp"] = np.array([h["box"], h["obj"], h["cls"], h["theta"], h["anchor_t"], 0.0], np.float32)
    rows = []
    for i, x in enumerate(p):
        g = x.grad.reshape(-1, 200)
        out[f"loss/gobj{i}"] = g[:, 4].numpy().copy()
        rest = g.clone()
        rest[:, 4] = 0
        r = torch.nonzero(rest.abs().sum(1) > 0).flatten()
        out[f"loss/grows{i}"] = r.numpy()
        out[f"loss/gvals{i}"] = g[r].numpy()
        rows.append(int(r.shape[0]))
    print("loss", float(loss), items.tolist(), "gradient rows per level", rows)
    assert all(rows), "every level needs matched rows"
    np.savez_compressed(HERE / "p6_golden.npz", **out)
    (HERE / "p6_ref_model_view.json").write_text(json.dumps(view, separators=(",", ":")) + "\n")


if __name__ == "__main__":
    main()
