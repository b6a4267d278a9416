"""Test-time-augmentation timing (dev tool): yolov5s and yolov5m (the calibrated benchmark models), B = 16, 1024^2 uint8 input.
Reports, as one JSON line, per model:
  plain_ms / tta_ms        CUDA-event mean per batch after warm-up of detect_records + non_max_suppression_obb, plain and
                           with augment=True, at conf_thres 0.01 (val.py: iou 0.4, multi-label, max_det 1500) and 0.25
                           (detect.py: iou 0.45, single label, max_det 1000)
  branch_ms                per TTA branch: the plan (branch 0 with its layout pass, branches 1-2 after their resample)
  resample_ms / _GBps      y5obb_scale_img_s2d_u8 per scaled branch, with its algorithmic bytes (one input read + the
                           stem-layout output)
  branch_gflop             per branch, summed from y5obb_conv_info; pruned_gflop: what the unpruned plans of the same shapes
                           would add (conv 21, C3 23 and the P5 Detect at scale 1, the P3 Detect at 0.67)
and the card's name and power limit, read in the same run.
python tools/time_tta.py [iters]"""
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from yolov5_obb_b200.engine import InferenceEngine  # noqa: E402
from yolov5_obb_b200.general import non_max_suppression_obb  # noqa: E402

B, S = 16, 1024
NMS = {"val": dict(conf_thres=0.01, iou_thres=0.4, multi_label=True, max_det=1500),
       "detect": dict(conf_thres=0.25, iou_thres=0.45, multi_label=False, max_det=1000)}


def event_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(size, x, iters, dev):
    m = bench.build_model(size, dev)
    out = {}
    for name, kw in NMS.items():
        out[f"plain_ms_{name}"] = round(event_ms(lambda: non_max_suppression_obb(m.detect_records(x), **kw), iters), 3)
        out[f"tta_ms_{name}"] = round(event_ms(lambda: non_max_suppression_obb(m.detect_records(x, augment=True), **kw),
                                               iters), 3)
    plan = m.tta_plan(tuple(x.shape), dev, compact_detect=True)
    e = plan.engines
    out["branch_ms"] = [round(event_ms(lambda: e[0].forward(x), iters), 3)] + \
        [round(event_ms(e[k].forward_s2d, iters), 3) for k in (1, 2)]
    rs = [event_ms(lambda k=k: plan.resample(x, k), 5 * iters) for k in (1, 2)]
    out["resample_ms"] = [round(t, 4) for t in rs]
    out["resample_bytes"] = [plan.resample_bytes(k, 1) for k in (1, 2)]
    out["resample_GBps"] = [round(plan.resample_bytes(k, 1) / t / 1e6, 1) for k, t in zip((1, 2), rs)]
    out["branch_gflop"] = [round(en.flops / 1e9, 1) for en in e]
    full = [m.records_plan(tuple(x.shape), dev).flops,
            InferenceEngine(m, B, plan.branches[2]["Hp"], plan.branches[2]["Wp"], dev, compact_detect=True).flops]
    out["pruned_gflop"] = [round((full[0] - e[0].flops) / 1e9, 1), round((full[1] - e[2].flops) / 1e9, 1)]
    out["rows_per_image"] = plan.rows_total
    del m, plan
    torch.cuda.empty_cache()
    return out


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    x = bench.synth_batch(B, 0).to(dev)
    res = {"card": card, "B": B, "S": S, "iters": iters, "input": "uint8"}
    for size in ("s", "m"):
        res[f"yolov5{size}"] = run(size, x, iters, dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
