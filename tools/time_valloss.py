"""Validation-loss timing (dev tool): yolov5s and yolov5m (the calibrated benchmark models) at 1024^2, B = 16 and 32, uint8
tiles, about 23 targets per tile.  Reports, as one JSON line, per model and batch:
  records_ms          CUDA-event mean per call after warm-up of Model.detect_records (the eval plan, compact records)
  records_loss_ms     detect_records + ComputeLoss.head_items (what Validator(compute_loss=...) adds per batch)
  head_items_ms       head_items alone, on the features of the last forward
  head_kernels_ms     the device time of head_items' kernels and memsets per call (torch.profiler, a separate loop): the
                      rest of head_items_ms is the host side of the call
  rows                matched rows (build_targets of the fp32 oracle on the same targets)
  head_bytes          algorithmic bytes of head_items: the Detect inputs read once, the obj logits written and read once,
                      the matched rows' features read and their logits written and read; head_GBps = head_bytes / head_items_ms
  materialised_bytes  the raw [B, 3, H, W, nc + 185] fp32 head output the loss would otherwise need, written once and read
                      once (its obj channel in 32-byte sectors plus the matched rows, as y5obb_loss_forward reads it)
and the card's name and power limit, read in the same run.
python tools/time_valloss.py [iters]"""
import json
import re
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from oracle import loss_ref  # noqa: E402
from tests.lossgen import synth_targets  # noqa: E402
from yolov5_obb_b200.loss import ComputeLoss  # noqa: E402

S = 1024


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


def run(m, B, iters, dev):
    x = bench.synth_batch(B, 0).to(dev)
    tg_cpu = torch.from_numpy(synth_targets(B, B * 23, S, nc=bench.NC, seed=3))
    tg = tg_cpu.to(dev)
    cl = ComputeLoss(m)
    plan = m.records_plan(tuple(x.shape), dev)
    out = {"nt": int(tg.shape[0])}
    out["records_ms"] = round(event_ms(lambda: m.detect_records(x), iters), 3)
    out["records_loss_ms"] = round(event_ms(lambda: (m.detect_records(x), cl.head_items(plan, tg)), iters), 3)
    m.detect_records(x)
    t = event_ms(lambda: cl.head_items(plan, tg), iters)
    out["head_items_ms"] = round(t, 4)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            cl.head_items(plan, tg)
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        if e.device_time_total > 0:
            k = re.search(r"(\w+)\(", e.key)
            name = k.group(1) if k else e.key[:40]
            per[name] = per.get(name, 0.0) + e.device_time_total / iters / 1e3
    out["head_kernels_ms"] = round(sum(per.values()), 4)
    out["head_kernels_top"] = {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:4]}
    det = m.model[-1]
    heads = plan.head_inputs()
    shapes = [torch.empty((B, det.na, s.H, s.W, det.no), device="meta") for s, _, _ in heads]
    _, _, idx, _, _ = loss_ref.build_targets(shapes, tg_cpu, det.anchors.cpu(), det.stride.cpu(), m.hyp["anchor_t"], det.na)
    rows = [int(i[0].numel()) for i in idx]
    cells = sum(B * det.na * s.H * s.W for s, _, _ in heads)
    feat = sum(B * s.H * s.W * s.C * 2 for s, _, _ in heads)
    row_bytes = sum(r * (s.C * 2 + 2 * det.no * 4) for r, (s, _, _) in zip(rows, heads))
    out["rows"] = rows
    out["head_bytes"] = feat + 2 * 4 * cells + row_bytes
    out["head_GBps"] = round(out["head_bytes"] / t / 1e6, 1)
    out["materialised_tensor_bytes"] = cells * det.no * 4
    out["materialised_bytes"] = cells * det.no * 4 + cells * 32 + sum(rows) * det.no * 4
    return out


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda:0")
    res = {"card": card, "S": S, "iters": iters, "input": "uint8"}
    for size in ("s", "m"):
        m = bench.build_model(size, dev)
        m.hyp = loss_ref.scaled_hyp(loss_ref.DEFAULT_HYP, 3, bench.NC, S)
        for B in (16, 32):
            res[f"yolov5{size}_B{B}"] = run(m, B, iters, dev)
        del m
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
