"""Golden vectors for the loss from the REFERENCE ComputeLoss (utils/loss.py, with the one-line clamp shim of
SURVEY §8(c)) and autograd on seeded inputs (tests/lossgen.py).  python tests/golden/make_loss_golden.py"""
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
from models.yolo import Model  # noqa: E402
from tests.lossgen import synth_preds, synth_targets  # noqa: E402

# in-memory source shim: torch >= 1.12 refuses clamp_ with a float tensor bound (loss.py:267)
src = (ref_import.REF / "utils" / "loss.py").read_text()
src = src.replace("gj.clamp_(0, feature_wh[1] - 1), gi.clamp_(0, feature_wh[0] - 1)",
                  "gj.clamp_(0, int(feature_wh[1]) - 1), gi.clamp_(0, int(feature_wh[0]) - 1)")
assert "int(feature_wh[1])" in src
mod = types.ModuleType("ref_loss")
mod.__dict__["__name__"] = "utils.loss_shimmed"
exec(compile(src, str(ref_import.REF / "utils" / "loss.py"), "exec"), mod.__dict__)


def main():
    out = {}
    hyp = yaml.safe_load((ref_import.REF / "data" / "hyps" / "obb" / "hyp.finetune_dota.yaml").read_text())
    from tests.losscases import CASES as cases
    for name, c in cases.items():
        torch.manual_seed(0)
        m = Model("models/yolov5n.yaml", ch=3, nc=15)
        h = dict(hyp)
        nl = 3
        h["box"] *= 3. / nl
        h["cls"] *= 15 / 80. * 3. / nl
        h["obj"] *= (c["imgsz"] / 640) ** 2 * 3. / nl
        h["theta"] *= 3. / nl
        h["label_smoothing"] = c.get("ls", 0.0)
        m.hyp = h
        cl = mod.ComputeLoss(m)
        p = [x.requires_grad_(True) for x in synth_preds(c["B"], c["imgsz"], seed=c["seed"])]
        tg = torch.from_numpy(synth_targets(c["B"], c["nt"], c["imgsz"], seed=c["seed"]))
        loss, items = cl(p, tg)
        (loss * 3.0).backward()  # upstream gradient 3.0 (what GradScaler would multiply in)
        out[f"{name}/targets"] = tg.numpy()
        out[f"{name}/loss"] = loss.detach().numpy()
        out[f"{name}/items"] = items.numpy()
        out[f"{name}/hyp"] = np.array([h["box"], h["obj"], h["cls"], h["theta"], h["anchor_t"], h["label_smoothing"]], np.float32)
        for i, x in enumerate(p):
            g = x.grad.reshape(-1, 200)
            out[f"{name}/gobj{i}"] = g[:, 4].numpy().copy()
            rest = g.clone()
            rest[:, 4] = 0
            rows = torch.nonzero(rest.abs().sum(1) > 0).flatten()
            out[f"{name}/grows{i}"] = rows.numpy()
            out[f"{name}/gvals{i}"] = g[rows].numpy()
        print(name, float(loss), items.tolist(), [int(out[f"{name}/grows{i}"].shape[0]) for i in range(3)])
    np.savez_compressed(HERE / "loss_golden.npz", **out)


if __name__ == "__main__":
    main()
