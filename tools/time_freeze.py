"""Training step with frozen layers (train.py --freeze): TrainStep.step and its backward plan for freeze [0], [10] and
[0, 1, 2], timed alternately in one process on one model per size (one training arena; the engine keeps one backward plan
per set of frozen layers).

Per (model, freeze): TrainStep.step median and range over `steps` steps after warm-up (host clock around a synchronised
step), the backward plan's device time (CUDA events around its graph replay), its launch steps and FLOPs, and the bytes of
activation-sized buffers it needs without an arena.  The card's name and power limit are read in the same run.  Prints one
JSON line.
usage: python tools/time_freeze.py [steps=20] [rounds=3] [B=16] [imgsz=1024] [sizes=s,m]"""
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from tests.lossgen import synth_targets
from tests.modelgen import build_mirror
from tests.tilegen import synth_tiles
from yolov5_obb_b200.train_step import TrainStep, freeze_layers

FREEZES = ([0], [10], [0, 1, 2])


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    B = int(sys.argv[3]) if len(sys.argv) > 3 else 16
    S = int(sys.argv[4]) if len(sys.argv) > 4 else 1024
    sizes = sys.argv[5].split(",") if len(sys.argv) > 5 else ["s", "m"]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    imgs = synth_tiles(B, S, seed=1).to(dev)
    tg = torch.from_numpy(synth_targets(B, 24 * B, S, nc=15, seed=2)).to(dev)
    out = dict(card=card, B=B, imgsz=S, steps=steps, rounds=rounds, results={})
    for size in sizes:
        m = build_mirror(size, nc=15, seed=0).train().to(dev)
        ts = TrainStep(m, batch_size=64, imgsz=S)   # (accumulate 1: every step ends with the fused optimizer step)
        m.reserve_train_arena(B, S, S, dev)
        times = {str(f): [] for f in FREEZES}
        for _ in range(rounds):
            for f in FREEZES:
                freeze_layers(m, f)
                for _ in range(3):                    # warm-up: plan switch, graph captures, fused table
                    ts.step(imgs, tg)
                torch.cuda.synchronize()
                for _ in range(steps):
                    t0 = time.perf_counter()
                    ts.step(imgs, tg)
                    torch.cuda.synchronize()
                    times[str(f)].append((time.perf_counter() - t0) * 1e3)
        eng = m._last_train_engine
        res = {}
        for f in FREEZES:
            freeze_layers(m, f)
            ts.step(imgs, tg)
            plan = eng._bwd
            G = [torch.randn(o.shape, device=dev) * 0.01 for o in eng.det_out]
            for _ in range(3):
                plan.run(G)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n = 20
            e0.record()
            for _ in range(n):
                plan.run(G)
            e1.record()
            torch.cuda.synchronize()
            t = times[str(f)]
            res[str(f)] = dict(step_ms_median=round(statistics.median(t), 3), step_ms_min=round(min(t), 3),
                               step_ms_max=round(max(t), 3), backward_ms=round(e0.elapsed_time(e1) / n, 3),
                               backward_steps=len(plan.steps), backward_gflop=round(plan.flops / 1e9, 1),
                               backward_buffer_mb=round(plan.nbytes / 2 ** 20, 1))
            print(f"yolov5{size} B{B} {S}x{S} freeze {f}: " + "  ".join(f"{k} {v}" for k, v in res[str(f)].items()),
                  flush=True)
        out["results"][f"yolov5{size}"] = res
        del ts, m, eng, plan
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
