"""Host logic of the fp16 inference plans: which models get them, how plans are keyed, what is refused, and the constants the
C ABI and the Python side share."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.modelgen import build_mirror
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.conv import F16, pack_weights
from yolov5_obb_b200.engine import plan_dtype
from yolov5_obb_b200.ensemble import Ensemble
from yolov5_obb_b200.general import DetectRecords, half_threshold

ROOT = Path(__file__).resolve().parents[1]


def test_a_half_model_plans_fp16_and_a_float_model_bf16():
    m = build_mirror("n", nc=15, seed=0)
    assert plan_dtype(m) == torch.bfloat16 and m._precision_key() == ()
    m.half()
    assert plan_dtype(m) == torch.float16 and m._precision_key() == ("f16",)
    m.float()
    assert plan_dtype(m) == torch.bfloat16


def test_mixed_parameter_dtypes_are_refused():
    m = build_mirror("n", nc=15, seed=0)
    m.model[0].half()
    with pytest.raises(RuntimeError, match="mixes parameter dtypes"):
        plan_dtype(m)


def test_ensemble_precision_follows_its_members():
    a, b = build_mirror("n", nc=15, seed=0), build_mirror("n", nc=15, seed=1)
    e = Ensemble([a, b])
    assert e._precision_key() == ()
    e.half()
    assert e._precision_key() == ("f16",)


def test_training_an_fp16_model_is_refused():
    m = build_mirror("n", nc=15, seed=0).half().train()
    with pytest.raises(RuntimeError, match="fp16 parameters"):
        m.forward_train(torch.zeros((1, 3, 64, 64), dtype=torch.float16))


def test_plans_are_keyed_by_precision():
    """The keys Model.records_plan / tta_plan / forward use: the bf16 keys are those of a float model, the fp16 ones carry
    the precision, so a process can hold both kinds."""
    m = build_mirror("n", nc=15, seed=0)
    key_bf = ("records", (1, 3, 64, 64), 0) + m._precision_key()
    m.half()
    key_fp = ("records", (1, 3, 64, 64), 0) + m._precision_key()
    assert key_bf == ("records", (1, 3, 64, 64), 0) and key_fp != key_bf


def test_half_threshold_rounds_through_fp32_to_fp16():
    for thr in (0.001, 0.01, 0.1, 0.25, 0.3, 0.45, 0.6, 1 / 3):
        assert half_threshold(thr) == float(np.float16(np.float32(thr)))
    assert half_threshold(0.25) == 0.25
    assert half_threshold(0.001) == 0.0010004043579101562


def test_detect_records_default_to_bf16_plans():
    d = torch.zeros((1, 4, 24))
    assert not DetectRecords(d, 15).half and DetectRecords(d, 15, True).half


def test_pack_weights_rounds_the_fused_fp32_weights_to_fp16():
    w = torch.randn(24, 16, 3, 3, generator=torch.Generator().manual_seed(0)) * 3
    b = torch.randn(24, generator=torch.Generator().manual_seed(1))
    wp, bp = pack_weights(w, b, dtype=torch.float16)
    assert wp.dtype == torch.float16 and bp.dtype == torch.float32
    assert torch.equal(wp[:, :24, :16], w.permute(2, 3, 0, 1).reshape(9, 24, 16).half())
    wb, _ = pack_weights(w, b)
    assert wb.dtype == torch.bfloat16


def test_header_and_python_constants_agree():
    h = (ROOT / "include" / "y5obb.h").read_text()
    assert int(re.search(r"#define Y5OBB_CONV_F16 (\d+)", h).group(1)) == F16
    assert int(re.search(r"#define Y5OBB_NMS_HALF (\d+)", h).group(1)) == _lib.NMS_HALF
    for name in ("y5obb_stem_s2d_f16", "y5obb_stem_s2d_u8_f16", "y5obb_scale_img_s2d_f16", "y5obb_scale_img_s2d_u8_f16",
                 "y5obb_sppf_pool_f16", "y5obb_letterbox_s2d_u8_f16", "y5obb_scene_tiles_s2d_u8_f16",
                 "y5obb_loss_forward_head_f16"):
        assert re.search(rf"\bint {name}\(", h), name

