"""Where a conv tile's cycles go, ops 0-49 of the benchmark's plan (dev tool): python tools/time_conv_epilogue.py

The plan is bench.py's: InferenceEngine(bench.build_model("s"), 16, 1024, 1024, compact_detect=True) on bench.synth_batch(16, 0).
The tool builds the library with -DY5OBB_CONV_PROBE
into build/conv_probe/ (apart from liby5obb.so) and runs each conv launch of the plan once on it, in a child process: thread 0
of every CTA sums clock64 cycles per phase of each of its first 64 tiles.  The phases are waiting for the first operands,
the MMAs, bias/SiLU staged, residual available and stores issued, plus the gap to the next tile.  Printed per op: mean cycles
per tile for each phase (over CTAs and tiles), then the means of each schedule class.  The probe's stamps cost cycles of their
own (the epilogue stamps each 64-column block), so compare phases within a build rather than against CUDA-event times.
The card's name, power limit and maximum SM clock are printed first.
"""
import argparse
import ctypes
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
PROBE_DIR = ROOT / "build" / "conv_probe"
PHASES = ["to tile", "wait operands", "MMA", "staged", "residual", "stores"]
LAST_OP = 49   # ops 0-49: every conv before the Detect head


def plans():
    """(label, engine, [(op index, Conv)]) for ops 0-49 of the bench's plan."""
    import bench
    from yolov5_obb_b200.engine import InferenceEngine
    m = bench.build_model(bench.MODEL).cuda()
    x = bench.synth_batch(bench.BATCH, 0).cuda()
    out = []
    for label, flags in (("default", 0),):
        eng = InferenceEngine(m, bench.BATCH, bench.IMG, bench.IMG, torch.device("cuda:0"), conv_flags=flags, compact_detect=True)
        for _ in range(3):
            eng.forward(x)
        torch.cuda.synchronize()
        conv_of = {id(c._h): c for c in eng.convs}
        ops = []
        for i, op in enumerate(eng.ops[:LAST_OP + 1]):
            d = op.__defaults__
            c = conv_of.get(id(d[0])) if d else None
            if c is not None:
                ops.append((i, c))
        out.append((label, eng, ops))
    return out


def sched_class(info):
    if info["ctas_per_sm"] == 2:
        return "2 CTAs/SM"
    return "1 CTA/SM, resident" if info["resident"] else "1 CTA/SM, streamed"


def probe_child(so):
    from yolov5_obb_b200 import _lib
    _lib._LIBPATH = Path(so)
    L = _lib.lib()
    dims = (ctypes.c_int * 3)()
    buf = np.zeros(264 * 64 * 6, dtype=np.int64)

    def read():
        _lib.check(L.y5obb_conv_probe(ctypes.c_void_p(buf.ctypes.data), ctypes.c_size_t(buf.nbytes), dims), "probe")
        return buf.reshape(dims[0], dims[1], dims[2]).copy()

    st = _lib.stream_ptr(torch.device("cuda:0"))
    print("phase cycles per tile (thread 0 of each CTA, its first 64 tiles; mean over CTAs and tiles)")
    hdr = f"{'op':>3} {'epilogue':>8} {'class':>18} {'tile_cyc':>8}  " + "  ".join(f"{p:>15}" for p in PHASES) + "  epi_frac"
    for label, eng, ops in plans():
        print(hdr)
        cls = {}
        for i, conv in ops:
            torch.cuda.synchronize()
            read()   # clears the stamps
            eng.ops[i](st)
            torch.cuda.synchronize()
            s = read().astype(np.float64)
            inf = conv.info()
            s = s[:inf["grid"]]
            ok = s[:, :, 2] > 0                 # tiles whose MMAs were stamped
            ok[:, 0] = False                    # the first tile has no "to tile" gap
            ph = s[ok]
            if ph.size == 0:
                print(f"{i:3d} {label:>8}  (no complete tiles stamped)")
                continue
            mean = ph.mean(0)
            tile = mean.sum()
            epi = mean[3:].sum() / tile
            c = sched_class(inf)
            cls.setdefault(c, []).append(mean)
            print(f"{i:3d} {label:>8} {c:>18} {tile:8.0f}  " + "  ".join(f"{v:7.0f} ({v / tile:4.0%})" for v in mean) +
                  f"  {epi:8.0%}")
        for c, ms in cls.items():
            mean = np.mean(ms, 0)
            tile = mean.sum()
            print(f"{'all':>3} {label:>8} {c:>18} {tile:8.0f}  " + "  ".join(f"{v:7.0f} ({v / tile:4.0%})" for v in mean) +
                  f"  {mean[3:].sum() / tile:8.0%}   ({len(ms)} ops)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--probe-child", metavar="SO", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.probe_child:
        probe_child(a.probe_child)
        return
    assert torch.cuda.is_available(), "time_conv_epilogue.py needs cuda:0"
    from time_detect import build_probe, card
    print(f"card: {card()}")
    so = build_probe("Y5OBB_CONV_PROBE", PROBE_DIR, "liby5obb_conv_probe.so")
    sys.stdout.flush()
    subprocess.run([sys.executable, str(Path(__file__).resolve()), "--probe-child", str(so)], check=True)


if __name__ == "__main__":
    main()
