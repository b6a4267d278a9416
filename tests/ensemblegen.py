"""Members and input of the ensemble golden, shared by tests/golden/make_ensemble_golden.py (run on the REFERENCE's
models/experimental.Ensemble) and the ensemble tests (run on yolov5_obb_b200.ensemble.Ensemble).

The members are yolov5n and yolov5n6 (nc=15, torch seed 0, tests/modelgen.seeded_state with the Detect obj / class rows
raised so that hundreds of rows pass the NMS threshold); the input is 2x3x128x192, a multiple of 64, so that the P5
member's 0.83 and 0.67 branches pad to multiples of 32 (128x160, 96x160) and the P6 member's to multiples of 64 (128x192,
128x192).  The golden stores the box columns and the sampled rows of tests/ttagen.pieces() (not the row sums, which the
tests do not read), and the reference's non_max_suppression_obb on the rows with NMS_KW."""
import torch

MEMBERS = ("n", "n6")
NC = 15
DET_KW = dict(obj_bias=1.0, cls_bias=-1.0, det_gain=6.0)
NMS_KW = dict(conf_thres=0.3, iou_thres=0.45, multi_label=True, max_det=300)


def ensemble_input():
    return torch.rand(2, 3, 128, 192, generator=torch.Generator().manual_seed(654))
