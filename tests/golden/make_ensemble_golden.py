"""Golden vectors of model ensembles from the REFERENCE (models/experimental.py Ensemble, eval, `ens(x)` and
`ens(x, augment=True)`; utils/general.py non_max_suppression_obb) — run in the authoring container:
    python tests/golden/make_ensemble_golden.py
Writes ensemble_golden.npz: for the members and input of tests/ensemblegen.py, per form ("plain", "tta") the ensemble's
rows [2, A, 200] as the box columns and sampled rows of tests/ttagen.pieces(), their shape, and per image the reference
NMS output [k, 7] with ensemblegen.NMS_KW."""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
from models.experimental import Ensemble  # noqa: E402  (the reference)
from models.yolo import Model  # noqa: E402
from utils.general import non_max_suppression_obb  # noqa: E402
from tests.ensemblegen import DET_KW, MEMBERS, NC, NMS_KW, ensemble_input  # noqa: E402
from tests.modelgen import seeded_state  # noqa: E402
from tests.ttagen import pieces  # noqa: E402


def ref_member(key):
    torch.manual_seed(0)
    cfg = f"models/hub/yolov5{key}.yaml" if key.endswith("6") else f"models/yolov5{key}.yaml"
    return seeded_state(Model(cfg, ch=3, nc=NC), 0, **DET_KW).eval()


def main():
    ens = Ensemble()
    for key in MEMBERS:
        ens.append(ref_member(key))
    ens.eval()
    x = ensemble_input()
    out = {"x_sum": np.float64(x.double().sum().item())}
    for form, augment in (("plain", False), ("tta", True)):
        with torch.no_grad():
            pred, none = ens(x, augment=augment)
        assert none is None
        for k, v in pieces(pred.numpy()).items():
            if k != "rowsum":
                out[f"{form}/{k}"] = v
        out[f"{form}/shape"] = np.array(pred.shape)
        dets = non_max_suppression_obb(pred.clone(), **NMS_KW)
        for b, d in enumerate(dets):
            out[f"{form}/nms/{b}"] = d.numpy()
        print(form, tuple(pred.shape), [tuple(d.shape) for d in dets])
    np.savez_compressed(HERE / "ensemble_golden.npz", **out)


if __name__ == "__main__":
    main()
