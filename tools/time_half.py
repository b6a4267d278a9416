"""Timing of the fp16 inference plans against the bf16 ones: python tools/time_half.py [--reps N]

For yolov5s and yolov5m (calibrated benchmark models, nc=15) at b16 1024^2, prints one JSON line: the card's name and power
limit (read in the same run), then per model the mean time of one detect_records + non_max_suppression_obb call of the bf16
plan (fp32 parameters) and of the fp16 plan (the same model after .half()): CUDA events around --reps calls after warm-up,
the two forms alternated three times (median of the three).  The outputs stay on the device."""
import argparse
import copy
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.modelgen import calibrated_bench_model  # noqa: E402
from tests.tilegen import synth_tiles  # noqa: E402
from tools.time_ensemble import card  # noqa: E402
from yolov5_obb_b200.general import non_max_suppression_obb  # noqa: E402

DEV = torch.device("cuda:0")
KW = dict(conf_thres=0.25, iou_thres=0.45, multi_label=True, max_det=1500)


def step_ms(model, x, reps):
    def once():
        non_max_suppression_obb(model.detect_records(x), return_packed="async", **KW)
    for _ in range(5):
        once()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        once()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    x = synth_tiles(16, 1024, seed=0).to(DEV)
    res = dict(card=card(), batch=16, size=1024)
    for size in ("s", "m"):
        m = calibrated_bench_model(size, nc=15)
        bf = m.to(DEV)
        fp = copy.deepcopy(m).half().to(DEV)
        t = {"bf16_ms": [], "fp16_ms": []}
        for _ in range(3):
            t["bf16_ms"].append(step_ms(bf, x, args.reps))
            t["fp16_ms"].append(step_ms(fp, x, args.reps))
        res[f"yolov5{size}"] = {k: round(statistics.median(v), 3) for k, v in t.items()}
        res[f"yolov5{size}"]["fp16_over_bf16"] = round(statistics.median(t["fp16_ms"]) / statistics.median(t["bf16_ms"]), 3)
        del bf, fp, m
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
