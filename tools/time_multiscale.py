"""Multi-scale training (TrainStep(multi_scale=True), train.py --multi-scale) at batch 16, imgsz 1024: prints ONE JSON line
per model with
  arena_bytes, peak_allocated      the reserved arena and torch.cuda.max_memory_allocated over the whole run
  outside_bytes                    per size: what each plan holds outside the arena (BN vectors, packed weights, graphs)
  first_visit_ms                   per size: plan build (TrainEngine + BackwardPlan), the eager step, the capturing step
  steady_ms                        at 512, 1024, 1536: the multi-scale step (graphs replayed) and a single-shape TrainStep
                                   on batches of that size, alternated in rounds; median and min-max spread of each
  resize                           per size: y5obb_scale_img_s2d_u8 time (CUDA events, median of 20) and algorithmic bytes
                                   (uint8 input read once, stem-layout output written once)
  run200_ms                        mean step time of 200 seeded multi-scale steps once every size has its graphs
and the card's name and power limit, read in the same run.
python tools/time_multiscale.py [models=s,m]"""
import copy
import json
import random
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests.lossgen import synth_targets  # noqa: E402
from tests.modelgen import build_mirror  # noqa: E402
from tests.tilegen import synth_tiles  # noqa: E402
from yolov5_obb_b200 import _lib, train_backward, train_engine  # noqa: E402
from yolov5_obb_b200.train_step import TrainStep  # noqa: E402

B, S, DEV = 16, 1024, "cuda:0"
SIZES = list(range(512, 1537, 32))


class _Sizes:
    def __init__(self, values):
        self.values = list(values)

    def randrange(self, lo, hi):
        return self.values.pop(0)


def _timed_init(cls, acc):
    init = cls.__init__

    def wrapped(self, *a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        init(self, *a, **k)
        torch.cuda.synchronize()
        acc.append((time.perf_counter() - t0) * 1e3)
    cls.__init__ = wrapped
    return init


def _step_ms(ts, imgs, tg):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ts.step(imgs, tg)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def _events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(n):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def _stat(v):
    return dict(median=round(statistics.median(v), 3), min=round(min(v), 3), max=round(max(v), 3))


def run(size):
    torch.cuda.reset_peak_memory_stats()
    m0 = build_mirror(size, nc=15, seed=0).train()
    m = copy.deepcopy(m0).to(DEV)
    imgs = synth_tiles(B, S, seed=1).to(DEV)
    tg = torch.from_numpy(synth_targets(B, 24 * B, S, nc=15, seed=2)).to(DEV)
    t0 = time.perf_counter()
    ts = TrainStep(m, batch_size=B, imgsz=S, multi_scale=True)
    reserve_ms = (time.perf_counter() - t0) * 1e3
    arena = m._train_arena
    builds = []
    saved = (_timed_init(train_engine.TrainEngine, builds), _timed_init(train_backward.BackwardPlan, builds))
    first = {}
    for s in SIZES:                    # visit 1: plan build + eager step; visit 2: graph capture
        ts.rng = _Sizes([s])
        builds.clear()
        eager = _step_ms(ts, imgs, tg)
        ts.rng = _Sizes([s])
        capture = _step_ms(ts, imgs, tg)
        first[s] = dict(build=round(sum(builds), 1), eager=round(eager - sum(builds), 1), capture=round(capture, 1))
    train_engine.TrainEngine.__init__, train_backward.BackwardPlan.__init__ = saved
    outside = {e.H: e.outside_bytes for k, e in m._engines.items() if k[0] == "train"}

    steady = {}
    for s in (512, 1024, 1536):
        ms_t, one_t = [], []
        try:
            m1 = copy.deepcopy(m0).to(DEV)
            one = TrainStep(m1, batch_size=B, imgsz=S)
            x1 = imgs if s == S else torch.nn.functional.interpolate(imgs.float(), size=(s, s), mode="bilinear",
                                                                      align_corners=False).round().clamp(0, 255).to(torch.uint8)
            t1 = tg.clone()
            t1[:, 2:6] *= s / S
            for _ in range(3):
                _step_ms(one, x1, t1)
        except torch.cuda.OutOfMemoryError:
            one = None
        for _ in range(5):
            for _ in range(4):
                ts.rng = _Sizes([s])
                ms_t.append(_step_ms(ts, imgs, tg))
            if one is not None:
                for _ in range(4):
                    one_t.append(_step_ms(one, x1, t1))
        steady[s] = dict(multi_scale=_stat(ms_t), single_shape=_stat(one_t) if one_t else "out of memory")
        one = m1 = None
        torch.cuda.empty_cache()

    L = _lib.lib()
    out = torch.empty((B, SIZES[-1] // 2, SIZES[-1] // 2 + 2, 16), dtype=torch.bfloat16, device=DEV)
    resize = {}
    for s in SIZES:
        if s == S:
            continue
        t = _events_ms(lambda: _lib.check(L.y5obb_scale_img_s2d_u8(imgs.data_ptr(), out.data_ptr(), B, S, S, s, s, s, s, 0,
                                                                     0.0, 1, _lib.stream_ptr()), "resize"), 20)
        nbytes = B * 3 * S * S + B * (s // 2) * (s // 2) * 32
        resize[s] = dict(ms=round(statistics.median(t), 4), bytes=nbytes, gbps=round(nbytes / statistics.median(t) / 1e6, 1))
    del out

    for s in SIZES:                    # visit 3: every size replays its graphs from here on
        ts.rng = _Sizes([s])
        ts.step(imgs, tg)
    ts.rng = random.Random(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(200):
        ts.step(imgs, tg)
    torch.cuda.synchronize()
    run200 = (time.perf_counter() - t0) * 1e3 / 200
    return dict(model=f"yolov5{size}", B=B, imgsz=S, reserve_ms=round(reserve_ms, 1), arena_bytes=arena.nbytes,
                peak_allocated=torch.cuda.max_memory_allocated(), outside_bytes=outside, first_visit_ms=first,
                steady_ms=steady, resize=resize, run200_ms=round(run200, 2))


def main():
    models = sys.argv[1].split(",") if len(sys.argv) > 1 else ["s", "m"]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    for size in models:
        print(json.dumps(dict(card=card, **run(size))), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
