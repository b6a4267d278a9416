"""Golden vectors of the validation loss from the REFERENCE model and ComputeLoss — run in the authoring container:
    python tests/golden/make_valloss_golden.py
For yolov5n and yolov5s (nc=15, torch seed 0, tests/modelgen.seeded_state with obj_bias tests/vallossgen.OBJ_BIAS) in eval
mode, over the batches of tests/vallossgen.batch: val.py's own loss lines, with the reference's ComputeLoss (utils/loss.py,
the clamp shim of make_loss_golden.py) and hyp.finetune_dota.yaml scaled as train.py:249-252 does:
    loss = torch.zeros(4)                                                       # val.py:179
    out, train_out = model(im)                                                  # val.py:195 (im = uint8 / 255, :186-187)
    loss += compute_loss([x.float() for x in train_out], targets)[1]           # val.py:198-199
    (loss.cpu() / len(dataloader)).tolist()                                     # val.py:333
Writes valloss_golden.npz: per size the per-batch items [N_BATCHES, 4] and the accumulated results [4]; per batch the targets
and the image sum (the tests regenerate the images from their seed and check the sum)."""
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
from tests.modelgen import seeded_state  # noqa: E402
from tests import vallossgen as VG  # noqa: E402

src = (ref_import.REF / "utils" / "loss.py").read_text()
src = src.replace("gj.clamp_(0, feature_wh[1] - 1), gi.clamp_(0, feature_wh[0] - 1)",
                  "gj.clamp_(0, int(feature_wh[1]) - 1), gi.clamp_(0, int(feature_wh[0]) - 1)")
assert "int(feature_wh[1])" in src
mod = types.ModuleType("ref_loss")
mod.__dict__["__name__"] = "utils.loss_shimmed"
exec(compile(src, str(ref_import.REF / "utils" / "loss.py"), "exec"), mod.__dict__)


def main():
    hyp = yaml.safe_load((ref_import.REF / "data" / "hyps" / "obb" / "hyp.finetune_dota.yaml").read_text())
    nl, nc = 3, 15
    hyp["box"] *= 3 / nl
    hyp["cls"] *= nc / 80 * 3 / nl
    hyp["obj"] *= (VG.HYP_IMGSZ / 640) ** 2 * 3 / nl
    hyp["theta"] *= 3 / nl
    hyp["label_smoothing"] = 0.0
    out = {"hyp": np.array([hyp["box"], hyp["obj"], hyp["cls"], hyp["theta"], hyp["anchor_t"]], np.float64)}
    batches = [VG.batch(i) for i in range(VG.N_BATCHES)]
    for i, (im, tg) in enumerate(batches):
        out[f"batch{i}/targets"] = tg.numpy()
        out[f"batch{i}/im_sum"] = np.int64(im.long().sum().item())
    for size in VG.SIZES:
        torch.manual_seed(0)
        m = Model(f"models/yolov5{size}.yaml", ch=3, nc=nc)
        seeded_state(m, 0, obj_bias=VG.OBJ_BIAS).eval()
        m.hyp = hyp
        compute_loss = mod.ComputeLoss(m)
        loss = torch.zeros(4)
        items = []
        with torch.no_grad():
            for im, tg in batches:
                x = im.float()
                x /= 255
                _, train_out = m(x)
                it = compute_loss([t.float() for t in train_out], tg)[1]
                items.append(it.numpy().copy())
                loss += it
        out[f"{size}/items"] = np.stack(items)
        out[f"{size}/results"] = np.array((loss.cpu() / len(batches)).tolist(), np.float64)
        print(size, out[f"{size}/items"].tolist(), out[f"{size}/results"].tolist())
    np.savez_compressed(HERE / "valloss_golden.npz", **out)


if __name__ == "__main__":
    main()
