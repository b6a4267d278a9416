"""Golden vectors of test-time augmentation from the REFERENCE model (models/yolo.py Model, `m(x, augment=True)`, eval) — run
in the authoring container:  python tests/golden/make_tta_golden.py
Writes tta_golden.npz: for yolov5n and yolov5s (nc=15, torch seed 0, tests/modelgen.seeded_state), the augmented output
[2, A_tta, 200] on tests/ttagen.tta_input(), stored as tests/ttagen.pieces() describes."""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import ref_import  # noqa: E402

ref_import.setup()
sys.path.insert(0, str(HERE.parents[1]))
from models.yolo import Model  # noqa: E402  (the reference)
from tests.modelgen import seeded_state  # noqa: E402
from tests.ttagen import pieces, tta_input  # noqa: E402


def main():
    x = tta_input()
    out = {"x_sum": np.float64(x.double().sum().item())}
    for size in ("n", "s"):
        torch.manual_seed(0)
        m = Model(f"models/yolov5{size}.yaml", ch=3, nc=15)
        seeded_state(m, 0).eval()
        with torch.no_grad():
            pred, none = m(x, augment=True)
        assert none is None
        for k, v in pieces(pred.numpy()).items():
            out[f"{size}/{k}"] = v
        out[f"{size}/shape"] = np.array(pred.shape)
        print(size, tuple(pred.shape), float(pred.abs().mean()))
    np.savez_compressed(HERE / "tta_golden.npz", **out)


if __name__ == "__main__":
    main()
