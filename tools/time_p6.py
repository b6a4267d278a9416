"""Timing of the four-level P6 models (models/hub/yolov5{s,m}6.yaml) beside yolov5s: python tools/time_p6.py [--reps N]

Prints one JSON line: the card's name and power limit (read in the same run), then per (model, image size), batch 16
  records_nms_ms   detect_records + non_max_suppression_obb on the calibrated benchmark model, CUDA events around
                   --reps calls after warm-up (mean per call);
  train_step_ms    TrainStep.step (fused SGD + EMA) on the same batch with 16 * 40 targets: host clock around a synchronised
                   step, median / min / max of --reps steps after warm-up;
the loss forward + backward at nl = 4 (yolov5s6 b16 1280^2 logits, CUDA events, mean), and the stride-64 layers of the
yolov5s6 b16 1280^2 and 1024^2 inference plans as tools/time_engine.py reports them: microseconds (median of --reps forwards),
algorithmic FLOP / bytes, the data-sheet bound and which peak sets it, and the grid against the card's SM count."""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.lossgen import synth_targets  # noqa: E402
from tests.modelgen import calibrated_bench_model  # noqa: E402
from tests.tilegen import synth_tiles  # noqa: E402
from yolov5_obb_b200 import _lib  # noqa: E402
from yolov5_obb_b200.engine import InferenceEngine  # noqa: E402
from yolov5_obb_b200.general import non_max_suppression_obb  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12   # H100 SXM data sheet: dense bf16, HBM3
DEV = torch.device("cuda:0")
B = 16


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


def records_nms(m, x, reps):
    def call():
        non_max_suppression_obb(m.detect_records(x), 0.25, 0.45, multi_label=True, max_det=1500)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    return events_ms(call, reps)


def train_step(m, x, reps):
    from yolov5_obb_b200.train_step import TrainStep
    m.train()
    ts = TrainStep(m, batch_size=64, imgsz=x.shape[2])
    tg = torch.from_numpy(synth_targets(B, 40 * B, x.shape[2], nc=15, seed=7)).to(DEV)
    for _ in range(3):
        ts.step(x, tg)
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        ts.step(x, tg)
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    m.eval()
    return dict(median=statistics.median(t), min=min(t), max=max(t))


def loss_fwd_bwd(m, x, reps):
    from yolov5_obb_b200.loss import ComputeLoss
    from yolov5_obb_b200.train_step import TrainStep
    m.train()
    ts = TrainStep(m, batch_size=64, imgsz=x.shape[2], ema=False)
    with torch.no_grad():
        p = [o.detach().clone().requires_grad_(True) for o in m(x)]
    m.eval()
    cl = ComputeLoss(m)
    assert cl.nl == 4 and ts.gs == 64
    tg = torch.from_numpy(synth_targets(B, 40 * B, x.shape[2], nc=15, seed=7)).to(DEV)

    def call():
        loss, _ = cl(p, tg)
        torch.autograd.grad(loss, p)
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    return events_ms(call, reps)


def stride64_layers(m, S, reps, n_sm):
    """tools/time_engine.py's per-op event timing, reported for the convs whose output is at stride 64."""
    eng = InferenceEngine(m, B, S, S, DEV, compact_detect=True)
    x = torch.rand(B, 3, S, S, device=DEV)
    for _ in range(3):
        eng.forward(x)
    torch.cuda.synchronize()
    st = _lib.stream_ptr(DEV)
    times = [[] for _ in eng.ops]
    for _ in range(reps):
        evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(eng.ops) + 1)]
        evs[0].record()
        for i, op in enumerate(eng.ops):
            op(st)
            evs[i + 1].record()
        torch.cuda.synchronize()
        for i in range(len(eng.ops)):
            times[i].append(evs[i].elapsed_time(evs[i + 1]))
    conv_of = {id(c._h): c for c in eng.convs}
    rows = []
    for i, op in enumerate(eng.ops):
        d = op.__defaults__
        conv = conv_of.get(id(d[0])) if d else None
        if conv is None:
            continue
        c = conv.desc
        ho = (c.Hin + 2 * c.pad_h - c.KH) // c.stride + 1
        if ho * 64 != S:
            continue
        inf = conv.info()
        tf, tb = inf["flops"] / PEAK_FLOPS, inf["hbm_bytes"] / PEAK_BYTES
        us = statistics.median(times[i]) * 1e3
        rows.append(dict(op=i, k=c.KH, stride=c.stride, cin=c.Cin, cout=c.Cout, out_hw=ho, us=round(us, 1),
                         gflop=round(inf["flops"] / 1e9, 2), mb=round(inf["hbm_bytes"] / 1e6, 1),
                         bound_us=round(max(tf, tb) * 1e6, 1), bound_by="flop" if tf >= tb else "hbm",
                         frac_of_bound=round(max(tf, tb) * 1e6 / us, 3), grid=inf["grid"], sms=n_sm,
                         ctas_per_sm=inf["ctas_per_sm"], block_n=inf["block_n"]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_p6.py measures on a CUDA device; none is visible")
    out = dict(card=card(), batch=B, reps=args.reps, runs=[])
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for size, S in (("s6", 1280), ("m6", 1280), ("s6", 1024), ("s", 1024)):
        m = calibrated_bench_model(size, nc=15, seed=0).to(DEV).eval()
        x = synth_tiles(B, S, seed=0).to(DEV)
        run = dict(model=f"yolov5{size}", img=S, records_nms_ms=round(records_nms(m, x, args.reps), 3))
        try:
            run["train_step_ms"] = {k: round(v, 2) for k, v in train_step(m, x, args.reps).items()}
        except torch.cuda.OutOfMemoryError:
            run["train_step_ms"] = "out of memory at batch 16"
        del m
        torch.cuda.empty_cache()
        out["runs"].append(run)
        print(json.dumps(run), file=sys.stderr, flush=True)
    m = calibrated_bench_model("s6", nc=15, seed=0).to(DEV).eval()
    x = synth_tiles(B, 1280, seed=0).to(DEV)
    out["loss_fwd_bwd_ms_nl4_s6_b16_1280"] = round(loss_fwd_bwd(m, x, args.reps), 3)
    m.invalidate()
    torch.cuda.empty_cache()
    out["stride64_layers"] = {f"yolov5s6 b16 {S}": stride64_layers(m, S, args.reps, n_sm) for S in (1280, 1024)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
