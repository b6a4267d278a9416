"""Times the Detect launches of the benchmark's plan (dev tool): python tools/time_detect.py [--probe] [--reps N]

The plan is bench.py's: InferenceEngine(bench.build_model("s"), 16, 1024, 1024, compact_detect=True) on bench.synth_batch(16, 0).
Each Detect launch (one per level) is timed alone with CUDA events, the median of --reps launches, for the records epilogue
and for the shared epilogue (Y5OBB_CONV_DETECT_GENERIC) in the same process.  Beside it: the launch's FLOP, the bytes the
records plan really moves (bf16 input + fp32 records; y5obb_conv_info's hbm_bytes counts a det_no-wide bf16 output instead)
and the bound max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s) from the H100 SXM data sheet.  The card's name, power limit and
maximum SM clock are printed first, because a power-limited card reaches less.

--probe also builds the library with -DY5OBB_DETECT_PROBE into build/detect_probe/ (apart from liby5obb.so) and runs the
same launches on it in a child process: thread 0 of every CTA stamps clock64 at each phase of its tiles, and the tool prints
how a tile's cycles split between waiting for the operands, the MMAs, the theta arg-max, staging and issuing the stores.
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
PROBE_DIR = ROOT / "build" / "detect_probe"
PHASES = ["wait operands", "MMA", "theta arg-max", "staging", "stores", "to next tile"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card name still comes from torch
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi: {e})"


def plans():
    """(label, engine, [(level, op index, ConvOp)]) for the records epilogue and the shared one, on the bench's input."""
    import bench
    from yolov5_obb_b200.conv import DETECT_GENERIC
    from yolov5_obb_b200.engine import InferenceEngine
    m = bench.build_model(bench.MODEL).cuda()
    x = bench.synth_batch(bench.BATCH, 0).cuda()
    out = []
    for label, flags in (("records", 0), ("generic", DETECT_GENERIC)):
        eng = InferenceEngine(m, bench.BATCH, bench.IMG, bench.IMG, torch.device("cuda:0"), conv_flags=flags, compact_detect=True)
        for _ in range(3):
            eng.forward(x)
        torch.cuda.synchronize()
        conv_of = {id(c._h): c for c in eng.convs}
        det = [(ly[1], i, conv_of[id(eng.ops[i].__defaults__[0])]) for i, ly in enumerate(eng.op_layers)
               if isinstance(ly, tuple) and ly[0] == "Detect"]
        out.append((label, eng, det))
    return out


def records_bound(eng, conv):
    d = conv.desc
    in_bytes = 2.0 * d.B * d.Hin * d.Win * d.Cin
    rec_bytes = 4.0 * d.B * (d.Cout // d.det_no) * d.Hin * d.Win * eng.rec_w
    flops = conv.info()["flops"]
    return flops, in_bytes + rec_bytes, max(flops / PEAK_FLOPS, (in_bytes + rec_bytes) / PEAK_BYTES)


def time_ops(reps):
    from yolov5_obb_b200 import _lib
    st = _lib.stream_ptr(torch.device("cuda:0"))
    res = {}
    for label, eng, det in plans():
        for lvl, i, conv in det:
            op = eng.ops[i]
            for _ in range(5):
                op(st)
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
            evs[0].record()
            for k in range(reps):
                op(st)
                evs[k + 1].record()
            torch.cuda.synchronize()
            us = statistics.median(evs[k].elapsed_time(evs[k + 1]) for k in range(reps)) * 1e3
            res.setdefault(lvl, {})[label] = (i, us, conv, eng)
    print(f"{'op':>3} {'level':>5} {'HxW':>9} {'K':>4} {'GFLOP':>6} {'MB':>6} {'bound_us':>8} {'generic_us':>10} "
          f"{'records_us':>10} {'speedup':>7} {'frac':>5}")
    tot = {"generic": 0.0, "records": 0.0}
    tot_bound = 0.0
    for lvl in sorted(res):
        i, us_new, conv, eng = res[lvl]["records"]
        us_old = res[lvl]["generic"][1]
        fl, by, bound = records_bound(eng, conv)
        tot["records"] += us_new
        tot["generic"] += us_old
        tot_bound += bound * 1e6
        d = conv.desc
        print(f"{i:3d} {'P%d' % (lvl + 3):>5} {'%dx%d' % (d.Hin, d.Win):>9} {d.Cin:4d} {fl / 1e9:6.1f} {by / 1e6:6.1f} "
              f"{bound * 1e6:8.1f} {us_old:10.1f} {us_new:10.1f} {us_old / us_new:7.2f} {bound * 1e6 / us_new:5.2f}")
    print(f"sum: generic {tot['generic']:.1f} us, records {tot['records']:.1f} us, bound {tot_bound:.1f} us")


def build_probe(define="Y5OBB_DETECT_PROBE", out_dir=PROBE_DIR, name="liby5obb_probe.so"):
    """liby5obb.so's sources compiled with -D`define` into out_dir/name (apart from liby5obb.so)."""
    from yolov5_obb_b200.build import CSRC, NVCC_FLAGS
    obj = out_dir / "obj"
    obj.mkdir(parents=True, exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))

    def cc(s):
        r = subprocess.run(["nvcc", *NVCC_FLAGS, f"-D{define}", "-c", str(s), "-o", str(obj / (s.stem + ".o"))],
                           capture_output=True, text=True)
        if r.returncode:
            raise RuntimeError(f"nvcc failed for {s.name}:\n{r.stdout}\n{r.stderr}")

    with ThreadPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        list(ex.map(cc, srcs))
    so = out_dir / name
    r = subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", str(so),
                        *[str(obj / (s.stem + ".o")) for s in srcs]], capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return so


def probe_child(so):
    from yolov5_obb_b200 import _lib
    _lib._LIBPATH = Path(so)
    L = _lib.lib()
    dims = (ctypes.c_int * 3)()
    buf = np.zeros(264 * 64 * 6, dtype=np.int64)

    def read():
        _lib.check(L.y5obb_detect_probe(ctypes.c_void_p(buf.ctypes.data), ctypes.c_size_t(buf.nbytes), dims), "probe")
        return buf.reshape(dims[0], dims[1], dims[2]).copy()

    st = _lib.stream_ptr(torch.device("cuda:0"))
    print(f"phase cycles per tile (thread 0 of each CTA, its first {64} tiles; mean over CTAs and tiles)")
    print(f"{'op':>3} {'epilogue':>8} {'tile_cyc':>8}  " + "  ".join(f"{p:>14}" for p in PHASES))
    for label, eng, det in plans():
        for lvl, i, conv in det:
            torch.cuda.synchronize()
            read()   # clears the stamps
            eng.ops[i](st)
            torch.cuda.synchronize()
            s = read().astype(np.float64)
            grid = conv.info()["grid"]
            s = s[:grid]
            ok = (s[:, :, 0] > 0) & (s[:, :, 5] > 0)
            ok[:, -1] = False
            ok[:, :-1] &= s[:, 1:, 0] > 0       # a next tile exists: the last phase runs to its start
            d = np.diff(s, axis=2)               # TILE->FULL, FULL->MMA, MMA->ARGMAX, ARGMAX->STAGED, STAGED->STORED
            nxt = np.zeros_like(s[:, :, 0])
            nxt[:, :-1] = s[:, 1:, 0] - s[:, :-1, 5]
            ph = np.concatenate([d, nxt[:, :, None]], 2)[ok]
            if ph.size == 0:
                print(f"{i:3d} {label:>8}  (no complete tiles stamped)")
                continue
            mean = ph.mean(0)
            tile = mean.sum()
            print(f"{i:3d} {label:>8} {tile:8.0f}  " + "  ".join(f"{v:7.0f} ({v / tile:4.0%})" for v in mean))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60)
    ap.add_argument("--probe", action="store_true", help="also build and run the clock64 phase probe")
    ap.add_argument("--probe-child", metavar="SO", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.probe_child:
        probe_child(a.probe_child)
        return
    assert torch.cuda.is_available(), "time_detect.py needs cuda:0"
    print(f"card: {card()}")
    time_ops(a.reps)
    if a.probe:
        so = build_probe()
        sys.stdout.flush()
        subprocess.run([sys.executable, str(Path(__file__).resolve()), "--probe-child", str(so)], check=True)


if __name__ == "__main__":
    main()
