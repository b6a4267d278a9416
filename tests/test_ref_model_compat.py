"""INTEGRATION.md B3: the engine plans a model from module class NAMES and a fixed set of attributes, so it accepts the
reference's own `models.yolo.Model` object as well as the mirror.  tests/golden/check_ref_model_compat.py builds the
reference's Model (n / s / m) and stores the engine's view of it, its strides and its parameter / state_dict names and shapes
in tests/golden/ref_model_view.json; here the mirror built from the same yaml must match that record attribute by attribute,
so its state_dict loads strictly into the reference's Model and back."""
import sys
from pathlib import Path

import json

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "tests" / "golden"))
from check_ref_model_compat import GOLDEN, SIZES, record  # noqa: E402


def test_engine_view_of_reference_model_equals_mirror():
    from yolov5_obb_b200.yolo import Model as MirrorModel
    golden = json.loads(GOLDEN.read_text())
    for size in SIZES:
        torch.manual_seed(0)
        mir = record(MirrorModel(f"yolov5{size}.yaml", ch=3, nc=15))
        ref = golden[size]
        assert len(mir["view"]) == len(ref["view"]), size
        for ra, rb in zip(ref["view"], mir["view"]):
            assert ra == rb, f"yolov5{size}: the engine would see\n  reference {ra}\n  mirror    {rb}"
        assert mir["stride"] == ref["stride"], size
        assert mir["params"] == ref["params"], size
        assert mir["state_dict"] == ref["state_dict"], size
