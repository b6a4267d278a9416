"""Per-op CUDA-event timing of one inference plan against its roofline (dev tool): python tools/time_engine.py s 16 1024

Each op is timed with CUDA events around it, the median over REPS forwards.  For a conv the line also gives its algorithmic
FLOP and HBM bytes (y5obb_conv_info), the bound max(FLOP / peak, bytes / HBM peak) and which of the two it is, the fraction
of that bound reached, and the launch plan: BN, BK, pipeline stages, resident weights, row-shift A stages, units per stage,
CTAs per SM and grid.  Peaks are the H100 SXM data-sheet figures (dense bf16 989 TFLOP/s, HBM3 3.35 TB/s); the card's name
and power limit are printed first, because a power-limited card reaches less.

Y5OBB_TE_CALIBRATED=1: the benchmark's model and batch (bench.build_model / bench.synth_batch).
Y5OBB_TE_RECORDS=1: the benchmark's plan (Detect rows as compact records).
Y5OBB_CONV_FLAGS: y5obb_conv_desc.flags for every layer (e.g. 64 = one CTA per SM everywhere).
"""
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tests.modelgen import build_mirror
from yolov5_obb_b200 import _lib
from yolov5_obb_b200.engine import InferenceEngine

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
REPS = int(os.environ.get("Y5OBB_TE_REPS", "20"))

size, B, S = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the card name still comes from torch
    smi = f"{torch.cuda.get_device_name(0)} (nvidia-smi: {e})"
print(f"card: {smi}")
if os.environ.get("Y5OBB_TE_CALIBRATED") == "1":   # the benchmark's 'alive' model (tests/modelgen.calibrated_bench_model)
    import bench
    m = bench.build_model(size).cuda()
    x = bench.synth_batch(B, 0).cuda()
else:
    m = build_mirror(size, nc=15, seed=0).cuda()
    x = None
eng = InferenceEngine(m, B, S, S, torch.device("cuda:0"), conv_flags=int(os.environ.get("Y5OBB_CONV_FLAGS", "0")),
                      compact_detect=os.environ.get("Y5OBB_TE_RECORDS") == "1")   # 1: the bench's plan (Detect rows as compact records)
if x is None:
    x = torch.rand(B, 3, S, S, device="cuda")
for _ in range(3):
    eng.forward(x)
torch.cuda.synchronize()
st = _lib.stream_ptr(eng.device)
times = [[] for _ in eng.ops]
for _ in range(REPS):
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(len(eng.ops) + 1)]
    evs[0].record()
    for i, op in enumerate(eng.ops):
        op(st)
        evs[i + 1].record()
    torch.cuda.synchronize()
    for i in range(len(eng.ops)):
        times[i].append(evs[i].elapsed_time(evs[i + 1]))

conv_of = {id(c._h): c for c in eng.convs}
print(f"{'op':>3} {'us':>8} {'GFLOP':>7} {'MB':>7} {'bound_us':>8} {'by':>4} {'frac':>5}  "
      f"{'BN':>3} {'BK':>3} {'st':>2} {'res':>3} {'rs':>2} {'grp':>3} {'cta':>3} {'grid':>4}")
tot = bound_tot = 0.0
for i, op in enumerate(eng.ops):
    ms = statistics.median(times[i])
    tot += ms
    d = op.__defaults__
    conv = conv_of.get(id(d[0])) if d else None
    if conv is None:
        print(f"{i:3d} {ms * 1000:8.1f}")
        continue
    inf = conv.info()
    tf, tb = inf["flops"] / PEAK_FLOPS, inf["hbm_bytes"] / PEAK_BYTES
    bound = max(tf, tb)
    bound_tot += bound
    g = lambda k: inf.get(k, "-")  # noqa: E731
    print(f"{i:3d} {ms * 1000:8.1f} {inf['flops'] / 1e9:7.1f} {inf['hbm_bytes'] / 1e6:7.1f} {bound * 1e6:8.1f} "
          f"{'flop' if tf >= tb else 'hbm':>4} {bound / (ms * 1e-3):5.2f}  {inf['block_n']:3d} {inf['block_k']:3d} "
          f"{inf['stages']:2d} {g('resident'):>3} {g('rowshift'):>2} {g('group'):>3} {g('ctas_per_sm'):>3} {inf['grid']:4d}")
print(f"sum of ops {tot:.3f} ms (convs' roofline bound {bound_tot * 1e3:.3f} ms); flops {eng.flops / 1e9:.1f} G -> "
      f"{eng.flops / tot / 1e9:.1f} TF/s; alg bytes {eng.hbm_bytes / 1e6:.0f} MB -> {eng.hbm_bytes / tot / 1e6:.0f} GB/s")
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
for _ in range(10):
    eng.forward(x)
e.record()
torch.cuda.synchronize()
print(f"forward {s.elapsed_time(e) / 10:.3f} ms -> {B / (s.elapsed_time(e) / 10) * 1000:.0f} img/s")
