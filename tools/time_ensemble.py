"""Timing of model ensembles (yolov5_obb_b200.ensemble.Ensemble): python tools/time_ensemble.py [--reps N] [--scene-reps N]

For yolov5s + yolov5m and yolov5s + yolov5s6 (calibrated benchmark models, nc=15) at 1024^2, prints one JSON line: the card's
name and power limit (read in the same run), then per pair
  ens_ms / members_ms   at b1 and b16: Ensemble.detect_records + one non_max_suppression_obb over the concatenated records,
                        beside the sum of each member's own detect_records + non_max_suppression_obb; CUDA events around
                        --reps calls after warm-up, mean per call, the two forms alternated three times (median of the three);
  scene                 SceneDetector.det on a 4000 x 4000 synthetic scene (25 tiles of 1056^2, or 1088^2 with the P6 member,
                        batch 16): host clock around synchronised calls, median of --scene-reps after one warm-up, and tiles/s.
The calls' outputs stay on the device; nothing is read back inside the timed windows."""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.modelgen import calibrated_bench_model  # noqa: E402
from tests.tilegen import synth_tiles  # noqa: E402
from yolov5_obb_b200.ensemble import Ensemble  # noqa: E402
from yolov5_obb_b200.general import non_max_suppression_obb  # noqa: E402
from yolov5_obb_b200.scene import SceneDetector  # noqa: E402

DEV = torch.device("cuda:0")
PAIRS = [("s", "m"), ("s", "s6")]
KW = dict(conf_thres=0.25, iou_thres=0.45, multi_label=True, max_det=1500)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (v.strip() for v in out.split(","))
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the name still comes from torch
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"not read ({e})")


def events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def pair_step(ens, x, reps):
    def ens_call():
        non_max_suppression_obb(ens.detect_records(x), **KW, return_packed="async")

    def members_call():
        for m in ens:
            non_max_suppression_obb(m.detect_records(x), **KW, return_packed="async")
    for _ in range(3):
        ens_call()
        members_call()
    torch.cuda.synchronize()
    a, b = [], []
    for _ in range(3):
        a.append(events_ms(ens_call, reps))
        b.append(events_ms(members_call, reps))
    return dict(ens_ms=round(statistics.median(a), 3), members_ms=round(statistics.median(b), 3),
                ens_runs=[round(v, 3) for v in a], members_runs=[round(v, 3) for v in b])


def scene(ens, reps):
    sc = synth_tiles(1, 4000, seed=11)[0].permute(1, 2, 0).contiguous().to(DEV)
    det = SceneDetector(ens, batch_size=16)
    det.det(sc)
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        det.det(sc)
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    ms = statistics.median(t) * 1e3
    return dict(tile=det.size, tiles=25, median_ms=round(ms, 2), min_ms=round(min(t) * 1e3, 2), tiles_per_s=round(25e3 / ms, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scene-reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_ensemble.py measures on a CUDA device; there is none here")
    out = dict(card=card())
    models = {k: calibrated_bench_model(k).to(DEV) for k in sorted({k for p in PAIRS for k in p})}
    for pair in PAIRS:
        ens = Ensemble([models[k] for k in pair])
        res = {}
        for B in (1, 16):
            x = synth_tiles(B, 1024, seed=3).to(DEV)
            res[f"b{B}"] = pair_step(ens, x, a.reps)
        res["scene"] = scene(ens, a.scene_reps)
        out["+".join(f"yolov5{k}" for k in pair)] = res
        ens.invalidate()
        for m in ens:
            m.invalidate()
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
