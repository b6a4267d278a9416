"""Validation-metric timing (dev tool) at DOTA-val scale: synthetic stats of `rows` detections (default 6M: several thousand
1024^2 tiles at conf_thres 0.01), 15 classes, 10 IoU thresholds, confidences on 1000 levels.  Reports the CUDA-event time of
ValStats.metrics() (ap_per_class + the one read + the numpy tail) and of the ValStats.add loop that accumulates the same rows
in batches of 16 x 1500, the host time of the CPU restatement oracle/valmetrics_ref.py on the first `cpu_rows` rows only
(labelled as such), and the card's name and power limit read in the same run.
python tools/time_val.py [rows] [cpu_rows] [reps]"""
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import valmetrics_ref as V  # noqa: E402
from yolov5_obb_b200.val import ValStats  # noqa: E402

NC, NIOU, B, MAX_DET = 15, 10, 16, 1500


def synth(rows, seed=0):
    rng = np.random.default_rng(seed)
    cls = rng.integers(0, NC, rows).astype(np.float32)
    conf = (rng.integers(10, 1001, rows) / 1000).astype(np.float32)
    tp = np.zeros((rows, NIOU), bool)
    tp[:, 0] = rng.random(rows) < 0.3 * conf
    for j in range(1, NIOU):
        tp[:, j] = tp[:, j - 1] & (rng.random(rows) < 0.85)
    n_l = np.bincount(cls.astype(np.int64)[tp[:, 0]], minlength=NC) + rng.integers(100, 1000, NC)
    tcls = np.repeat(np.arange(NC, dtype=np.float64), n_l)
    return tp, conf, cls, tcls


def main():
    rows = int(sys.argv[1]) if len(sys.argv) > 1 else 6_000_000
    cpu_rows = int(sys.argv[2]) if len(sys.argv) > 2 else 200_000
    reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    tp, conf, cls, tcls = synth(rows)
    per = B * MAX_DET
    nb = (rows + per - 1) // per
    dets = torch.zeros((nb * B, MAX_DET, 7), dtype=torch.float32)
    flat = dets.view(-1, 7)
    flat[:rows, 5], flat[:rows, 6] = torch.from_numpy(conf), torch.from_numpy(cls)
    correct = torch.zeros((nb * B * MAX_DET, NIOU), dtype=torch.bool)
    correct[:rows] = torch.from_numpy(tp)
    dets, correct = dets.to(dev), correct.view(nb * B, MAX_DET, NIOU).to(dev)
    counts = torch.full((nb * B,), MAX_DET, dtype=torch.int64)
    counts.view(-1)[-1] = MAX_DET - (nb * per - rows)
    counts = counts.to(dev)
    targets = torch.stack([torch.zeros(len(tcls)), torch.from_numpy(tcls).float()], 1).to(dev)
    empty = torch.zeros((0, 2), dtype=torch.float32, device=dev)

    def accumulate():
        vs = ValStats(NC, NIOU, dev)
        for i in range(nb):
            s = slice(i * B, (i + 1) * B)
            vs.add(dets[s], counts[s], correct[s], targets if i == 0 else empty)
        return vs

    out = {"card": card, "rows": rows, "classes": NC, "niou": NIOU, "batches": nb, "batch": f"{B}x{MAX_DET}"}
    for _ in range(2):
        vs = accumulate()
        m = vs.metrics()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        vs = accumulate()
    ev[1].record()
    torch.cuda.synchronize()
    out["device_add_loop_ms"] = round(ev[0].elapsed_time(ev[1]) / reps, 3)
    t = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = vs.metrics()
        t.append(time.perf_counter() - t0)
    out["device_metrics_ms"] = round(1e3 * float(np.median(t)), 3)
    out["map50"], out["map"] = float(m.results[2]), float(m.results[3])

    t0 = time.perf_counter()
    want = V.val_metrics([tp[:cpu_rows], conf[:cpu_rows], cls[:cpu_rows], tcls], NC)
    out["cpu_subset_rows"] = cpu_rows
    out["cpu_restatement_subset_ms"] = round(1e3 * (time.perf_counter() - t0), 1)
    vs = ValStats(NC, NIOU, dev)
    k = (cpu_rows + MAX_DET - 1) // MAX_DET
    sub = counts[:k].clone()
    sub[-1] = cpu_rows - (k - 1) * MAX_DET
    vs.add(dets[:k], sub, correct[:k], targets)
    assert np.array_equal(np.array(vs.metrics().results), np.array(want["results"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
